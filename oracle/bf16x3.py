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
    """(act(acc + bias) + residual) * out_scale [+ prev] in fp64, and its exactness record.  The order is the kernels'
    (``epilogue_f32`` states it step by step in fp32), but fp64 equals their fp32 result only where every step is
    exact, which the record guards: on grid data, with power-of-two slopes and scales.  tanh is never exact here."""
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


def _operands(a, bf16x3):
    """hi / lo parts of the fp32 operand a: its bf16 split, or (a, 0) for the FFMA engine"""
    return split(a) if bf16x3 else (a.float(), torch.zeros_like(a, dtype=torch.float32))


def conv1d_acc(x, w, *, stride=1, padding=(0, 0), dilation=1, groups=1, pad_mode="zero", pre_slope=1.0, lolo=False,
               bf16x3=True):
    """fp64 accumulator of the bf16x3 conv: sum of x_hi w_hi + x_lo w_hi + x_hi w_lo over (channel, tap) of
    lrelu(x, pre_slope) padded by ``padding`` = (left, right) in ``pad_mode`` (zero / reflect / replicate).
    ``lolo`` adds the x_lo w_lo term the tensor cores drop (then the result is the fp64 conv of the fp32 operands);
    ``bf16x3`` False: the FFMA engine's exact products of the fp32 operands.
    Returns (acc, per-element sum of the magnitudes of the terms, their grid)."""
    xh, xl = _operands(lrelu(x, pre_slope), bf16x3)
    wh, wl = _operands(w, bf16x3)
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


def conv_transpose1d_acc(x, w, *, stride, padding=0, output_padding=0, pre_slope=1.0, bf16x3=True):
    """fp64 accumulator of ConvTranspose1d (w: (cin, cout, k)) on lrelu(x) with bf16x3 (or, ``bf16x3`` False, exact
    fp32) products.  Returns (acc, per-element sum of the magnitudes of the terms, their grid)."""
    xh, xl = (t.double() for t in _operands(lrelu(x, pre_slope), bf16x3))
    wh, wl = (t.double() for t in _operands(w, bf16x3))
    kw = dict(stride=stride, padding=padding, output_padding=output_padding)
    acc = F.conv_transpose1d(xh, wh, **kw) + F.conv_transpose1d(xl, wh, **kw) + F.conv_transpose1d(xh, wl, **kw)
    bound = F.conv_transpose1d(xh.abs() + xl.abs(), wh.abs() + wl.abs(), **kw)
    return acc, bound, _term_grid(xh, xl, wh, wl)


def conv_transpose1d(x, w, bias=None, *, stride, padding=0, output_padding=0, pre_slope=1.0):
    """ConvTranspose1d (w: (cin, cout, k)) on lrelu(x) with bf16x3 products, + bias.  Returns (y fp32, Exactness)."""
    acc, bound, g = conv_transpose1d_acc(x, w, stride=stride, padding=padding, output_padding=output_padding,
                                         pre_slope=pre_slope)
    return _epilogue(acc, bound, g, bias, None, 1.0, None, 1.0, None)


def conv1d_wgrad_acc(x, gy, kernel, *, pad_left=0, dilation=1, groups=1, x_slope=1.0, g_slope=1.0):
    """fp64 accumulator of ``conv1d_wgrad``: (dw, per-element sum of the magnitudes of the terms, their grid)"""
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
    return acc, bound, _term_grid(gh, gl, xh, xl)


def conv1d_wgrad(x, gy, kernel, *, pad_left=0, dilation=1, groups=1, x_slope=1.0, g_slope=1.0):
    """Weight gradient of a stride-1 zero-padded conv: dw[co, ci, k] = sum_{b,t} gy'[b, co, t] x'[b, ci, t + k*D - pad]
    with gy' = lrelu(gy, g_slope), x' = lrelu(x, x_slope) and bf16x3 products gy_hi x_hi + gy_lo x_hi + gy_hi x_lo.
    Returns (dw fp32 (cout, cin / groups, kernel), Exactness)."""
    acc, bound, g = conv1d_wgrad_acc(x, gy, kernel, pad_left=pad_left, dilation=dilation, groups=groups, x_slope=x_slope,
                                     g_slope=g_slope)
    return _epilogue(acc, bound, g, None, None, 1.0, None, 1.0, None)


def resblock_pair(x, w1, b1, w2, b2, *, kernel_size, dilation, slope, out_scale=1.0, prev=None):
    """One HiFi-GAN ResBlock conv pair: h = conv_{k,d}(lrelu(x)) + b1 (exact in fp32 by its own guard), then
    y = [prev +] out_scale * (conv_{k,1}(lrelu(h)) + b2 + x), conv2 on split(lrelu(h)).  Returns (y, Exactness of both)."""
    k, d = kernel_size, dilation
    h, ex1 = conv1d(x, w1, b1, padding=(k - 1) // 2 * d, dilation=d, pre_slope=slope)
    y, ex2 = conv1d(h, w2, b2, padding=(k - 1) // 2, pre_slope=slope, residual=x, out_scale=out_scale, prev=prev)
    return y, ex1 & ex2


# ---------------------------------------------------------------------------------------------------- WaveNet layer
# Both tensor-core forms of the WaveNet residual layer (residual_block.py:102-140):
#   g  = conv_{K,d}(x) + W_aux c [+ b]    bf16x3, one fp32 accumulation (the aux 1x1 is extra K chunks)
#   z  = tanh(g[:H]) * sigmoid(g[H:])     the only inexact step: ex2.approx / div.approx (fused form, gate_fast) or
#                                         tanhf / __expf (two-launch form, the pre_gate producer)
#   so = bf16x3(split(z)) . [W_skip ; W_out]
#   skips (+)= so[:S] + b_skip ;  x' = (so[S:] + b_out + x) * fl32(sqrt(1/2))
# The fused form adds the conv bias inside the gate (one fma into the ex2 argument), reads x as its packed x_hi + x_lo
# and writes x' split into packed hi / lo words.
SQRT_HALF = float(np.float32(math.sqrt(0.5)))     # `rs` / `out_scale` of both forms
LOG2E2 = float(np.float32(2.8853900817779268))    # gate_fast: a-half factor 2 log2(e) in fp32
NLOG2E = float(np.float32(-1.4426950408889634))   # gate_fast: b-half factor -log2(e) in fp32
CLAMP_A = float(np.float32(43.28))                # gate_fast: clamp of the a-half ex2 argument
U32 = 2.0 ** -24                                   # unit roundoff of fp32 round to nearest
U_BF16 = 2.0 ** -8                                 # unit roundoff of bf16 round to nearest


def gate_fp64(a, b):
    """tanh(a) * sigmoid(b) in fp64"""
    a, b = a.double(), b.double()
    return torch.tanh(a) * torch.sigmoid(b)


# Gate inputs on which the device gate is exactly known (the identities that tests/test_gpu_wavenet_exact.py reads back
# on the device).  fused: gate_fast(0, .) = 0, gate_fast(-64, 128) = -1, gate_fast(-64, 0) = -0.5;
# two-launch: tanhf(0) = 0, tanhf(+-20) = +-1, sigmoidf_(20) = 1, sigmoidf_(0) = 0.5, sigmoidf_(-100) = 0.
EXACT_TANH = {"fused": {0.0: 0.0, -64.0: -1.0}, "two": {0.0: 0.0, 20.0: 1.0, -20.0: -1.0}}
EXACT_SIGMOID = {"fused": {0.0: 0.5, 128.0: 1.0}, "two": {20.0: 1.0, 0.0: 0.5, -100.0: 0.0}}


def gate_table(form):
    """The gate of ``form`` ("fused" / "two") on its exact classes: a function (a, b) -> z (fp64) that raises when an
    element is outside the table.  In the fused form a = 0 gives z = 0 for any b (ex2(0) - 1 = 0)."""
    ta, sg = EXACT_TANH[form], EXACT_SIGMOID[form]

    def gate(a, b):
        a, b = a.double(), b.double()
        za = torch.full_like(a, math.nan)
        sb = torch.full_like(b, math.nan)
        for k, v in ta.items():
            za[a == k] = v
        for k, v in sg.items():
            sb[b == k] = v
        z = za * sb
        if form == "fused":
            z[a == 0] = 0.0
        assert not torch.isnan(z).any(), f"gate input outside the exact {form} classes"
        return z

    return gate


def _same_pad(k, d):
    p = (k - 1) // 2 * d
    return (p, p)


def _bf16x3_acc(a, w, kw, drop_lo_hi=False, lolo=False):
    """fp64 sum of a_hi w_hi + a_lo w_hi + a_hi w_lo (F.conv1d with ``kw``), its magnitude bound and grid;
    ``drop_lo_hi`` leaves out a_lo w_hi, ``lolo`` adds a_lo w_lo"""
    ah, al = (t.double() for t in split(a))
    wh, wl = (t.double() for t in split(w))
    acc = F.conv1d(ah, wh, **kw) + F.conv1d(ah, wl, **kw)
    if not drop_lo_hi:
        acc = acc + F.conv1d(al, wh, **kw)
    if lolo:
        acc = acc + F.conv1d(al, wl, **kw)
    bound = F.conv1d(ah.abs() + al.abs(), wh.abs() + wl.abs(), **kw)
    return acc, bound, _term_grid(ah, al, wh, wl)


@dataclass
class WaveNetResult:
    """One emulated layer: fp32 g (two-launch: with the conv bias; fused: the accumulator, without it), z (fp64, the
    gate's value before the split), skips, x' and, for the fused form, xw = x' split as the kernel writes it (hi + lo
    values, fp32); an Exactness record per stage: ex_g (conv + aux [+ bias]), ex_skip, ex_x."""

    g: torch.Tensor
    z: torch.Tensor
    skips: torch.Tensor
    x: torch.Tensor
    xw: torch.Tensor
    ex_g: Exactness
    ex_skip: Exactness
    ex_x: Exactness

    @property
    def ex(self):
        return self.ex_g & self.ex_skip & self.ex_x


def wavenet_layer(x, c, w_conv, b_conv, w_aux, w_skip, b_skip, w_out, b_out, *, dilation, form, gate=None, skips=None,
                  skips_init=False, drop=(), lolo=False):
    """fp64 emulation of one WaveNet layer in the kernels' order, ``form`` "two" (pwgb_wavenet_layer_forward: two
    conv1d_tc launches) or "fused" (pwgb_wnstack_layer_forward).  Shapes: x (B, R, T), c (B, A, T) or None, w_conv
    (G, R, K), w_aux (G, A[, 1]), w_skip (S, H[, 1]), w_out (R, H[, 1]), biases 1-D or None, skips (B, S, T) or None
    (zeros).  ``gate(a, b)`` -> z in fp64 (default: tanh * sigmoid in fp64, rounded to fp32 as the kernels hold z);
    a and b include the conv bias.  The two-launch form always accumulates into skips; the fused form overwrites them
    when ``skips_init``.  ``drop`` names terms to leave out, to emulate broken kernels: "x_lo_w_hi" (conv),
    "z_lo_w_hi" (skip / out), "x_lo" (the fused residual reads x_hi only).  ``lolo`` adds both dropped lo*lo terms."""
    assert form in ("two", "fused")
    B, R, T = x.shape
    G, _, K = w_conv.shape
    H = G // 2
    S = w_skip.shape[0]
    acc, bound, g_grid = _bf16x3_acc(x, w_conv, dict(padding=_same_pad(K, dilation)[0], dilation=dilation),
                                     "x_lo_w_hi" in drop, lolo)
    if c is not None:
        a2, b2, gg2 = _bf16x3_acc(c, w_aux.reshape(G, -1, 1), {}, False, lolo)
        acc, bound, g_grid = acc + a2, bound + b2, min(g_grid, gg2)
    if form == "two":
        g32, ex_g = _epilogue(acc, bound, g_grid, b_conv, None, 1.0, None, 1.0, None)
        a, b = g32[:, :H].double(), g32[:, H:].double()
    else:
        g32, ex_g = _epilogue(acc, bound, g_grid, None, None, 1.0, None, 1.0, None)
        bc = torch.zeros(G, dtype=torch.float64) if b_conv is None else b_conv.double()
        a = g32[:, :H].double() + bc[:H].reshape(1, -1, 1)
        b = g32[:, H:].double() + bc[H:].reshape(1, -1, 1)
    z = gate_fp64(a, b).float().double() if gate is None else gate(a, b)
    w_so = torch.cat([w_skip.reshape(S, H), w_out.reshape(R, H)]).reshape(S + R, H, 1)
    so, so_bound, so_grid = _bf16x3_acc(z.float(), w_so, {}, "z_lo_w_hi" in drop, lolo)
    bso = None if b_skip is None else torch.cat([b_skip.reshape(-1), b_out.reshape(-1)])
    b_s, b_o = (None, None) if bso is None else (bso[:S], bso[S:])
    prev = None if (form == "fused" and skips_init) else (torch.zeros(B, S, T) if skips is None else skips)
    sk, ex_skip = _epilogue(so[:, :S], so_bound[:, :S], so_grid, b_s, None, 1.0, None, 1.0, prev)
    if form == "fused":
        xh, xl = split(x)
        res = xh.double() if "x_lo" in drop else xh.double() + xl.double()
    else:
        res = x
    xo, ex_x = _epilogue(so[:, S:], so_bound[:, S:], so_grid, b_o, None, 1.0, res, SQRT_HALF, None)
    hi, lo = split(xo)
    return WaveNetResult(g32, z, sk, xo, hi + lo, ex_g, ex_skip, ex_x)


def pack_words(x, halo, t_pad):
    """The packed hi / lo image of fp32 x (B, C, T) that wn_pack_kernel / wn_first_conv_kernel write: int32 words of
    [B][hi|lo][ceil(C/8)][t_pad][8 ch] bf16 (two channels per word, the even one in the low half), samples in rows
    [halo, halo + T), every other row and every channel >= C zero.  Returned flat, as the device buffer."""
    B, Cc, T = x.shape
    ng = (Cc + 7) // 8
    if B == 0:
        return torch.zeros(0, dtype=torch.int32)
    hi, lo = split(x)
    img = torch.zeros(B, 2, ng * 8, t_pad, dtype=torch.bfloat16)
    img[:, 0, :Cc, halo:halo + T] = hi.to(torch.bfloat16)
    img[:, 1, :Cc, halo:halo + T] = lo.to(torch.bfloat16)
    img = img.reshape(B, 2, ng, 8, t_pad).permute(0, 1, 2, 4, 3).contiguous()
    return img.view(torch.int16).view(torch.int32).reshape(-1)


def unpack_words(words, B, Cc, halo, t_pad, T):
    """inverse of pack_words: hi + lo of rows [halo, halo + T) as fp32 (B, Cc, T)"""
    ng = (Cc + 7) // 8
    if B == 0:
        return torch.zeros(0, Cc, T)
    img = words.reshape(-1).view(torch.int16).view(torch.bfloat16).reshape(B, 2, ng, t_pad, 8).float()
    v = img[:, 0] + img[:, 1]
    return v.permute(0, 1, 3, 2).reshape(B, ng * 8, t_pad)[:, :Cc, halo:halo + T].contiguous()


def fits_split(t):
    """every value survives the hi / lo split: hi + lo == t"""
    hi, lo = split(t)
    return bool(torch.equal(hi + lo, t.float()))


def zero_target_data(gen, B, R, G, S, T, K, dilation, *, lo_on="x", scale_w=2.0 ** -3, max_tries=64):
    """Data on which g == 0 exactly: W_aux = -I (A = G) and c = the bf16x3 conv of x, so the conditioning 1x1 cancels
    the conv at every element.  x and W_conv are grid values with lo parts on ``lo_on`` ("x" or "w") only; b_conv = 0
    (the fused kernel folds it into the ex2 argument); W_skip / W_out / b_skip / b_out / prior skips are grid values.
    Every c must survive the hi / lo split (c is fed through it); data that do not are redrawn from the same generator.
    Returns a dict of the layer's inputs."""
    for _ in range(max_tries):
        x = grid_values((B, R, T), gen, 1.0, hmax=1, lo=lo_on == "x")
        w = grid_values((G, R, K), gen, scale_w, hmax=1, lo=lo_on == "w")
        acc, bound, g = _bf16x3_acc(x, w, dict(padding=_same_pad(K, dilation)[0], dilation=dilation))
        c = acc.float()
        if not (torch.equal(c.double(), acc) and fits_split(c) and Exactness(float(bound.max()), g).ok):
            continue
        return dict(x=x, c=c, w_conv=w, b_conv=None, w_aux=-torch.eye(G), **_so_data(gen, R, G, S, B, T))
    raise AssertionError("zero_target_data: no draw survives the split")


def _so_data(gen, R, G, S, B, T):
    H = G // 2
    return dict(w_skip=grid_values((S, H), gen, 2.0 ** -2, hmax=3), w_out=grid_values((R, H), gen, 2.0 ** -2, hmax=3),
                b_skip=grid_values((S,), gen, 2.0 ** -1, hmax=3), b_out=grid_values((R,), gen, 2.0 ** -1, hmax=3),
                skips=grid_values((B, S, T), gen, 1.0, hmax=3))


def saturated_data(gen, B, R, G, S, T, form):
    """Data on which every gate input is in an exact class of ``form`` (EXACT_TANH / EXACT_SIGMOID): W_conv = 0,
    W_aux = I (A = G), b_conv = 0 and c drawn from the classes, so z is exactly 0, +-0.5 or +-1 (fused: 0, -0.5, -1).
    x, W_skip / W_out, the biases and prior skips are grid values.  Returns a dict of the layer's inputs."""
    H = G // 2
    ka = torch.tensor(sorted(EXACT_TANH[form]))
    kb = torch.tensor(sorted(EXACT_SIGMOID[form]))
    c = torch.cat([ka[torch.randint(0, len(ka), (B, H, T), generator=gen)],
                   kb[torch.randint(0, len(kb), (B, H, T), generator=gen)]], 1).float()
    assert fits_split(c)
    x = grid_values((B, R, T), gen, 1.0, hmax=3)
    return dict(x=x, c=c, w_conv=torch.zeros(G, R, 3), b_conv=None, w_aux=torch.eye(G), **_so_data(gen, R, G, S, B, T))


def bound_data(gen, B, R, G, S, A, T, K=3, hmax=2):
    """Bound-regime data (fused form): grid x, c, W_conv, W_aux and a nonzero grid conv bias, so that g is exact and
    spreads over the whole gate range, saturation included.  W_skip / W_out are readout weights: one nonzero power of
    two per row, so that the skip / out contraction is exact for any z and gate_bound isolates the gate."""
    H = G // 2

    def readout(n):
        w = torch.zeros(n, H)
        h = torch.randint(0, H, (n,), generator=gen)
        s = torch.randint(0, 2, (n,), generator=gen) * 2 - 1
        e = torch.randint(0, 4, (n,), generator=gen)
        w[torch.arange(n), h] = s.float() * torch.exp2(e.float())
        return w

    x = grid_values((B, R, T), gen, 1.0, hmax=hmax)
    c = grid_values((B, A, T), gen, 1.0, hmax=hmax)
    return dict(x=x, c=c, w_conv=grid_values((G, R, K), gen, 2.0 ** -3, hmax=hmax),
                b_conv=grid_values((G,), gen, 2.0 ** -1, hmax=3), w_aux=grid_values((G, A), gen, 2.0 ** -3, hmax=hmax),
                w_skip=readout(S), w_out=readout(R), b_skip=grid_values((S,), gen, 2.0 ** -3, hmax=1, zero_frac=0.5),
                b_out=grid_values((R,), gen, 2.0 ** -1, hmax=3),
                skips=grid_values((B, S, T), gen, 2.0 ** -3, hmax=1, zero_frac=0.5))


EPS_EX2 = 2.0 ** -22   # ex2.approx.ftz.f32: relative error budget
EPS_DIV = 2.0 ** -22   # __fdividef (div.approx): 2 ulp for 2^-126 <= |d| <= 2^126


def gate_fast_bound(ga, gb, ba, bb):
    """Per-element bound on |gate_fast(ga, gb) - tanh(ga + ba) sigmoid(gb + bb)| for the fused kernel's gate
    (wavenet_tc.cu: z = (Ea - 1) / ((Ea + 1)(1 + Eb)), Ea = ex2(min(pa, 43.28)), Eb = ex2(pb)), from these per-step
    budgets:
      - the ex2 arguments pa = RN(fma(ga, fl(2 log2 e), RN(ba fl(2 log2 e)))) (pb the same with -log2 e) differ from
        the exact 2 log2(e) a by (|ga| + |ba|) |fl(2 log2 e) - 2 log2 e|, plus one fp32 rounding of the bias product and
        one of the fma (2^-24 of their magnitudes);
      - ex2.approx has relative error EPS_EX2 and an argument error dp scales its result by 2^dp, so the device's Ea lies
        in Ea (1 +- rho_a), rho_a = (2^(|dp|) - 1) + EPS_EX2 (times 1.01 for the product of the two), Eb likewise;
      - t = (Ea - 1) / (Ea + 1) and s = 1 / (1 + Eb) are monotone in Ea and Eb, so the exact t s over those intervals
        is bounded by the corner values (this keeps the correlated error of Ea in numerator and denominator exact);
      - N = Ea - 1, D1 = Ea + 1, D2 = 1 + Eb and D = D1 D2 round once each to fp32.  A rounding is at most 2^-24 of
        its result, and at most the distance to an fp32 candidate: Ea (or 1) is one, so N and D1 move by at most 1 and
        D2 by at most Eb.  Relative: min(2^-24, 1 / |N|) + min(2^-24, 1 / D1) + min(2^-24, Eb / D2) + 2^-24, and the
        quotient costs EPS_DIV;
      - the clamp at 43.28 replaces tanh by t(2^43.28): that difference is computed exactly;
      - ftz: an ex2 result below 2^-126 is 0 (an absolute 2^-118 where pa < -120);
      - where D may exceed 2^125, __fdividef may return 0 (and ex2 may overflow): there the bound is |z| + 2^-100.
    Inputs: fp64 tensors of the accumulator halves (ga, gb, without bias) and the conv bias halves (ba, bb) broadcast
    to them."""
    ga, gb, ba, bb = (t.double() for t in (ga, gb, ba, bb))
    a, b = ga + ba, gb + bb
    z = gate_fp64(a, b)
    ln2 = math.log(2.0)

    def arg_err(g, bias, cf, c):
        pb_ = bias * cf
        return (g.abs() + bias.abs()) * abs(cf - c) + U32 * pb_.abs() + U32 * (g * cf + pb_).abs()

    c1, c2 = 2.0 / ln2, -1.0 / ln2
    pa = torch.clamp(c1 * a, max=CLAMP_A)
    pb = c2 * b
    ea, eb = torch.exp2(pa), torch.exp2(torch.clamp(pb, max=1000.0))
    ra = (torch.exp2(arg_err(ga, ba, LOG2E2, c1)) - 1 + EPS_EX2) * 1.01
    rb = (torch.exp2(arg_err(gb, bb, NLOG2E, c2)) - 1 + EPS_EX2) * 1.01

    def t_of(e):
        return (e - 1) / (e + 1)

    def s_of(e):
        return 1 / (1 + e)

    ts = [t_of(ea * (1 - ra)), t_of(ea * (1 + ra))]
    ss = [s_of(eb * (1 - rb)), s_of(eb * (1 + rb))]
    ideal = t_of(ea) * s_of(eb)
    corner = torch.stack([(t * s - ideal).abs() for t in ts for s in ss]).amax(0)
    mag = torch.stack([(t * s).abs() for t in ts for s in ss]).amax(0)
    ea_lo = ea * (1 - ra)
    rnd = (torch.clamp(1 / (ea_lo - 1).abs(), max=U32) + torch.clamp(1 / (ea_lo + 1), max=U32)
           + torch.clamp(eb * (1 + rb) / (1 + eb), max=U32) + U32 + EPS_DIV)
    e = corner + mag * rnd * 1.01 + (z - ideal).abs() + 2.0 ** -50 * z.abs() + 2.0 ** -100
    e = e + torch.where(pa < -120, torch.full_like(e, 2.0 ** -118), torch.zeros_like(e))
    huge = ((ea + 1) * (1 + eb) > 2.0 ** 125) | (pb > 125)
    return torch.where(huge, z.abs() + 2.0 ** -100, e)


def split_bound(v, e):
    """bound on |hi(w) + lo(w) - v| for any fp32 w with |w - v| <= e: |w - hi(w)| <= |v - hi(v)| + e (hi(w) is the
    bf16 nearest to w), lo rounds that remainder to 8 bits"""
    v = v.double()
    vh = v.float().to(torch.bfloat16).double()
    return e + U_BF16 * ((v - vh).abs() + e)


def gate_bound(d, dilation):
    """Per-element bounds (skips, x') of the fused layer on bound_data ``d`` (readout W_skip / W_out, skips_init False)
    against the fp64 layer with exact gate: skips_ref = w z + b_skip + skips, x'_ref = ((w z + b_out) + x) fl(sqrt 1/2).
    Derivation, per element:
      - g is exact (guarded), so the gate input error is the gate's own: e_z = gate_fast_bound;
      - the kernel contracts split(z_dev): |hi + lo - z| <= e_S = split_bound(z, e_z);
      - one nonzero power-of-two weight per row: so = w (hi + lo) exactly, error |w| e_S;
      - every later fp32 operation (+ b, + prior skips / + x_hi, + x_lo, * rs) adds at most 2^-24 of its result's
        magnitude (reference magnitude plus the error so far), an addition also at most its exact addend (zero biases
        and prior skips, which bound_data draws often, add nothing);
      - x' is written split: compare hi + lo of the words, split_bound again.
    Returns (bound_skips, bound_x, ref_skips, ref_x) as fp64 tensors."""
    x, c, w_conv, b_conv, w_aux = d["x"], d["c"], d["w_conv"], d["b_conv"], d["w_aux"]
    G, R, K = w_conv.shape
    H = G // 2
    S = d["w_skip"].shape[0]
    emu = wavenet_layer(x, c, w_conv, b_conv, w_aux, d["w_skip"], d["b_skip"], d["w_out"], d["b_out"], dilation=dilation,
                        form="fused", gate=gate_fp64, skips=d["skips"])
    emu.ex_g.check("gate_bound: g")
    for w in (d["w_skip"], d["w_out"]):
        nz = (w != 0).sum(1)
        assert bool((nz == 1).all()), "gate_bound needs one nonzero weight per row"
        m, _ = torch.frexp(w[w != 0])
        assert bool((m.abs() == 0.5).all()), "gate_bound needs power-of-two readout weights"
    g = emu.g.double()
    bc = b_conv.double().reshape(1, -1, 1)
    e_z = gate_fast_bound(g[:, :H], g[:, H:], bc[:, :H].expand_as(g[:, :H]), bc[:, H:].expand_as(g[:, H:]))
    z = emu.z
    e_s = split_bound(z, e_z)
    W = torch.cat([d["w_skip"], d["w_out"]]).double()
    so = torch.einsum("nh,bht->bnt", W, z)
    e_so = torch.einsum("nh,bht->bnt", W.abs(), e_s)

    def add(v, e, t):
        """v + t in fp32 (v an fp32 value within e of the reference, t exact): value, error.  The rounding is at most
        2^-24 of the result and at most |t| (v itself is a candidate)."""
        r = v + t
        return r, e + torch.minimum(U32 * (r.abs() + e), t.abs().expand_as(r))

    bs, bo = d["b_skip"].double().reshape(1, -1, 1), d["b_out"].double().reshape(1, -1, 1)
    v, e = add(so[:, :S], e_so[:, :S], bs)
    sk, e_sk = add(v, e, d["skips"].double())
    xh, xl = (t.double() for t in split(x))
    v, e = add(so[:, S:], e_so[:, S:], bo)
    v, e = add(v, e, xh)
    v, e = add(v, e, xl)
    xo = v * SQRT_HALF
    e = e * SQRT_HALF + U32 * (xo.abs() + e * SQRT_HALF)
    return e_sk, split_bound(xo, e), sk, xo


# ---------------------------------------------------------------------------------------------------- rounding on fp32
# The grid data above make every rounding exact, so they cannot see how a kernel rounds.  Here the operands are
# arbitrary fp32 values and the weights (or the activations) are one-hot: every output element then receives exactly
# one non-zero (activation, weight) pair, its terms a_hi w_hi + a_lo w_hi + a_hi w_lo with one operand equal to 1.0
# (hi = 1, lo = 0), so the accumulator is hi + lo of the other operand.  hi + lo spans at most 17 bits: it is exact in
# fp32, whatever the order of the (zero) other terms.  The epilogue that follows then has one correct fp32 result for
# each element, ``epilogue_f32``.  On random data the same emulation gives the value the bound ``conv_bound`` is
# centred on.
U_TC = 2.0 ** -23   # tensor-core accumulation: not specified as round-to-nearest (it aligns and truncates), one ulp
U_FFMA = 2.0 ** -24  # fp32 fma / add, round to nearest
SUBNORMAL = 2.0 ** -149  # absolute floor of one fp32 rounding (the subnormal spacing)
BF16_INF_FROM = 0x7F7F8000  # the smallest fp32 magnitude (bits) whose bf16 round to nearest is inf


def from_bits(u):
    """fp32 tensor with the bit patterns of the uint32 numpy array ``u``"""
    return torch.from_numpy(np.ascontiguousarray(u, dtype=np.uint32).view(np.float32).copy())


def fp32_values(shape, seed, special=False):
    """Arbitrary fp32 values, each element of one class drawn at random, both signs throughout:
      - "near": random bits with magnitudes in [2^-4, 2^4) (the classes the epilogue mixes most);
      - "bits": random bit patterns over every normal exponent, below ``BF16_INF_FROM``;
      - "tie": exact bf16 ties (low 16 bits 0x8000), the kept bit of either parity;
      - "lo_tie": hi + r with r an exact bf16 tie of the remainder (the lo part's own rounding);
      - "zero" (+-0) and "sub" (subnormals, which the build does not flush);
    ``special`` adds "huge" (magnitudes from ``BF16_INF_FROM`` to FLT_MAX, where hi rounds to inf), +-inf and NaN."""
    rng = np.random.default_rng(seed)
    n = int(np.prod(shape))
    classes = ["near"] * 6 + ["bits"] * 3 + ["tie"] * 2 + ["lo_tie"] * 2 + ["zero", "sub"]
    if special:
        classes += ["huge", "huge", "inf", "nan"]
    cls = rng.integers(0, len(classes), n)
    sign = rng.integers(0, 2, n).astype(np.uint32) << 31
    mant = rng.integers(0, 1 << 23, n, dtype=np.uint32)
    out = np.zeros(n, dtype=np.uint32)
    for i, c in enumerate(classes):
        m = cls == i
        k = int(m.sum())
        if c == "near":
            e = rng.integers(127 - 4, 127 + 4, k).astype(np.uint32)
            out[m] = (e << 23) | mant[m]
        elif c == "bits":
            e = rng.integers(1, 255, k).astype(np.uint32)
            out[m] = np.minimum((e << 23) | mant[m], BF16_INF_FROM - 1)
        elif c == "tie":
            e = rng.integers(127 - 20, 127 + 20, k).astype(np.uint32)
            out[m] = (e << 23) | (mant[m] & ~np.uint32(0xFFFF)) | 0x8000
        elif c == "lo_tie":
            # hi = 1.m7 * 2^E, r = +-(q + 1/2) 2^(E-16), q in [128, 256): |r| < 2^(E-8) (hi is its bf16), r is a tie
            e = rng.integers(-20, 20, k)
            hi = (1.0 + rng.integers(0, 128, k) / 128.0) * np.exp2(e)
            q = rng.integers(128, 256, k)
            r = (q + 0.5) * np.exp2(e - 16.0) * np.where(rng.integers(0, 2, k) == 1, 1.0, -1.0)
            out[m] = (hi + r).astype(np.float32).view(np.uint32)
        elif c == "zero":
            out[m] = 0
        elif c == "sub":
            out[m] = np.maximum(mant[m], 1)
        elif c == "huge":
            out[m] = rng.integers(BF16_INF_FROM, 0x7F7FFFFF, k, endpoint=True, dtype=np.uint32)
        elif c == "inf":
            out[m] = 0x7F800000
        else:
            out[m] = 0x7FC00000
    out |= sign
    return from_bits(out).reshape(shape)


def onehot_weight(cout, cin_g, K, offset=0):
    """the activation probe: w[co, (co + offset) % cin_g, co % K] = 1, every other weight 0 (each column reads one
    tap); with cout / groups < cin_g, the offsets of ``probe_offsets`` read every input channel between them"""
    w = torch.zeros(cout, cin_g, K)
    co = torch.arange(cout)
    w[co, (co + offset) % cin_g, co % K] = 1.0
    return w


def onehot_weight_transposed(cin, cout, K, stride):
    """the activation probe of a conv-transpose (w: (cin, cout, K)): for every column co and phase ph < stride one
    tap k = ph (mod stride) reads channel (co * stride + ph) % cin.  An output row meets the taps of one phase only, so
    it still reads one non-zero weight, and cout * stride >= cin columns-and-phases read every input channel."""
    w = torch.zeros(cin, cout, K)
    for ph in range(stride):
        taps = list(range(ph, K, stride))
        if not taps:
            continue
        for co in range(cout):
            w[(co * stride + ph) % cin, co, taps[co % len(taps)]] = 1.0
    return w


def onehot_positions(T, spacing, margin):
    """the time steps ``onehot_input`` sets"""
    return range(margin, T - margin, spacing)


def onehot_input(B, cin, T, spacing, margin, groups=1, offset=0):
    """the weight probe: x[b, g cin_g + ci, s] = 1 at s = margin + j * spacing, ci = (j + offset) mod cin_g, 0
    elsewhere.  With spacing beyond the conv's receptive field every output reads at most one of them, through one
    tap.  Where fewer steps than cin_g fit, the offsets of ``probe_offsets`` reach the other channels."""
    x = torch.zeros(B, cin, T)
    cin_g = cin // groups
    for j, s in enumerate(onehot_positions(T, spacing, margin)):
        for g in range(groups):
            x[:, g * cin_g + (j + offset) % cin_g, s] = 1.0
    return x


def probe_offsets(per_launch, channels):
    """channel offsets of the launches a probe needs when one launch reads ``per_launch`` consecutive channels of
    ``channels``: every channel is read by one of them"""
    return list(range(0, channels, per_launch)) if 0 < per_launch < channels else [0]


def pair_count(op, x, w):
    """the largest number of non-zero (operand, weight) pairs that reach one output element of ``op(x, w)`` (an fp64
    conv of the non-zero indicators): a one-hot probe is exact when it is at most 1"""
    return float(op((x != 0).double(), (w != 0).double()).max()) if x.numel() and w.numel() else 0.0


def conv1d_acc_ieee(x, w, *, padding, dilation=1, groups=1, pad_mode="zero", pre_slope=1.0, bf16x3=True):
    """The accumulator of a stride-1 conv with every term formed as the hardware forms it, non-finite values included
    (0 * inf = NaN, inf - inf = NaN): an explicit fp64 sum over (channel, tap), for small shapes.  Exact for one-hot
    probes; ``bf16x3`` False is the FFMA engine (fp32 operands, no split)."""
    a = lrelu(x, pre_slope)
    a = _pad(a, padding[0], padding[1], pad_mode)
    cout, cin_g, K = w.shape
    B, cin, Tp = a.shape
    t_out = Tp - (K - 1) * dilation
    win = torch.stack([a[..., k * dilation:k * dilation + t_out] for k in range(K)], -1)  # (B, cin, t_out, K)
    win = win.reshape(B, groups, cin_g, t_out, K)
    wg = w.reshape(groups, cout // groups, cin_g, K)
    with np.errstate(invalid="ignore", over="ignore"):
        if bf16x3:
            ah, al = (t.double().numpy() for t in split(win))
            wh, wl = (t.double().numpy() for t in split(wg))
            acc = (np.einsum("bgctk,gock->bgot", ah, wh) + np.einsum("bgctk,gock->bgot", al, wh)
                   + np.einsum("bgctk,gock->bgot", ah, wl))
        else:
            acc = np.einsum("bgctk,gock->bgot", win.double().numpy(), wg.double().numpy())
    return torch.from_numpy(acc).reshape(B, cout, t_out)


def epilogue_f32(acc, bias=None, post_act=None, post_slope=0.0, residual=None, out_scale=1.0, prev=None, *, tanh=None,
                 err=None):
    """The conv epilogue of every engine, step by step in fp32 (numpy float32, one rounding per step):
        v = acc + bias (0 without a bias);  v = act(v);  v = v + residual;  v = v * out_scale;  v = v + prev
    -- epi_store and the staged epilogue of conv1d_tc.cu (the staged accumulate is the bulk copy's fp32 add into y),
    the FFMA epilogue of conv1d_simt.cu, and conv2 of the fused ResBlock pair (residual = x); conv1 of the pair stops
    after the bias.  ``acc`` (fp64 or fp32) is rounded to fp32 first, a zero as +0.  act: "lrelu" v > 0 ? v : v * slope, "tanh"
    ``tanh(v)`` when given (the device's values, to check the other steps around it), else tanh in fp64 rounded to fp32.
    With ``err`` (per-element bound on |device accumulator - acc|) also returns the bound on |device output - result|:
    each step adds its input error times the step's slope and two roundings, 2^-24 of its result (device and
    emulation) plus the subnormal spacing; tanh adds libdevice's 2 ulp.  Returns y (fp32 tensor) [, bound fp64]."""
    f = np.float32
    a64 = acc.double().numpy()
    v = a64.astype(f) + f(0.0)  # every engine's accumulator starts at +0: a zero accumulator is +0
    shape = (1, -1) + (1,) * (v.ndim - 2)
    e = None if err is None else err.double().numpy() + np.abs(v.astype(np.float64) - a64)

    def rnd(q, e_in):
        """error after rounding a step whose exact result is q (fp64) from inputs within e_in"""
        return e_in * (1 + U_FFMA) + 2 * U_FFMA * np.abs(q) + SUBNORMAL

    with np.errstate(invalid="ignore", over="ignore"):
        if bias is not None:
            b = bias.float().numpy().reshape(shape)
            if e is not None:
                e = rnd(v.astype(np.float64) + b, e)
            v = v + b
        else:
            v = v + f(0.0)
        if post_act == "lrelu":
            s = f(post_slope)
            if e is not None:
                e = np.where(v > 0, e, rnd(v.astype(np.float64) * float(s), e))
            v = np.where(v > 0, v, v * s)
        elif post_act == "tanh":
            t = np.tanh(v.astype(np.float64)).astype(f) if tanh is None else np.asarray(tanh, dtype=f)
            if e is not None:
                e = e + 2.0 ** -22 * (np.abs(t) + e) + U_FFMA * np.abs(t) + SUBNORMAL
            v = t
        elif post_act not in (None, "none"):
            raise ValueError(post_act)
        if residual is not None:
            r = residual.float().numpy()
            if e is not None:
                e = rnd(v.astype(np.float64) + r, e)
            v = v + r
        s = f(out_scale)
        if e is not None:
            e = rnd(v.astype(np.float64) * float(s), e * float(s))
        v = v * s
        if prev is not None:
            p = prev.float().numpy()
            if e is not None:
                e = rnd(v.astype(np.float64) + p, e)
            v = v + p
    y = torch.from_numpy(np.ascontiguousarray(v, dtype=f))
    return y if e is None else (y, torch.from_numpy(e))


def accumulation_bound(mag, n, u):
    """gamma_{n-1} sum|terms| with gamma_m = m u / (1 - m u) (+ 2^-52 of it for the fp64 reference sum): the worst
    error of any order of n - 1 additions, each rounding by at most u of its result (Higham, Accuracy and Stability
    of Numerical Algorithms, 2nd ed., section 4.2)"""
    m = (n - 1) * u
    assert m < 0.5, "accumulation_bound: the sum is too long for the bound"
    return mag * (m / (1 - m) + 2.0 ** -52)
