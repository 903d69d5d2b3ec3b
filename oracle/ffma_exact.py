"""Exact fp64 reference of the plain-fp32 (FFMA) kernels, and the data on which their fp32 result is unique.

The FFMA engine (conv1d_simt.cu, the FFMA branch of convtr1d.cu, backward.cu, upsample.cu, s2d.cu, the pooling of
reduce.cu) multiplies fp32 operands and accumulates in fp32 (the bias gradient and the filter adjoint carry their long
sums in double).  As in oracle/bf16x3.py, when every product and every partial sum is an integer multiple of one power
of two g and stays below 2^22 g, each fp32 operation is exact and the correct output is unique: a kernel must
reproduce it bit for bit whatever order it sums in.  Every function here computes in float64 on the fp32 operands,
applies the epilogue in the kernel's order and returns ``(fp32 result, Exactness)``.

Data rules (the GPU tests follow them):
- one operand of every product carries a lo part (``grid_values(..., lo=True)``: 12 significant bits), the other is
  drawn with ``lo=False``; a kernel that rounded an operand to TF32 or bf16 would change the result.  Both assignments
  are covered.  The guard takes the grid of the actual products, grid(x) * grid(w): with lo parts on both operands the
  lo x lo products collapse it and the guard fails;
- slopes and scales are powers of two (0.5, 0.125);
- average-pool gradients are multiples of 12, so that gy / div is exact for every divisor 1 to 4;
- reductions over B * t_out (weight gradients) need sparse data to pass the guard; the sums that the kernels carry in
  double (bias gradient, filter adjoint) are exact below 2^52 grid steps and are rounded once to fp32, so long rows
  need no sparse data there.

CPU only."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from .bf16x3 import EXACT_BITS, Exactness, _epilogue, grid, grid_values, lrelu  # noqa: F401  (grid_values re-exported)

DOUBLE_BITS = 52  # sums carried in double: exact below 2^52 grid steps


def _double_exactness(bound, g):
    """a sum carried in double, on the scale of Exactness (whose guard is 2^EXACT_BITS grid steps)"""
    return Exactness(float(bound), math.ldexp(g, DOUBLE_BITS - EXACT_BITS))


def _values_exactness(*ts):
    """every element of the fp64 tensors is an fp32 value with at most EXACT_BITS significant bits (per element)"""
    worst = 0.0
    for t in ts:
        v = t.double().reshape(-1).numpy()
        v = np.abs(v[v != 0])
        if v.size == 0:
            continue
        m, e = np.frexp(v)
        n = np.ldexp(m, 53).astype(np.int64)
        low = np.log2((n & -n).astype(np.float64))
        worst = max(worst, float((53 - low).max()))  # significant bits of each element
    return Exactness(math.ldexp(1.0, int(worst)) if worst else 0.0, 2.0)


def _pad(x, left, right, mode):
    """rows padded by (left, right) in ``mode``; a negative right crops"""
    if right < 0:
        x = x[..., :x.shape[-1] + right]
        right = 0
    if mode in ("zero", "zeros"):
        return F.pad(x, (left, right))
    return F.pad(x, (left, right), mode=mode)


def columns(x, period):
    """(B, C, L) flat (or (B, C, rows, P)) -> (B * P, C, rows): the columns of the period view, L reflect-extended to
    rows * P (hifigan.py:365-369; the kernels' t_valid)"""
    B, Cc = x.shape[:2]
    x = x.reshape(B, Cc, -1)
    L = x.shape[-1]
    rows = -(-L // period)
    if rows * period > L:
        x = F.pad(x, (0, rows * period - L), mode="reflect")
    return x.reshape(B, Cc, rows, period).permute(0, 3, 1, 2).reshape(B * period, Cc, rows)


def uncolumns(y, B, period):
    """(B * P, C, t) -> (B, C, t, P), or (B, C, t) for P = 1"""
    y = y.reshape(B, period, *y.shape[1:]).permute(0, 2, 3, 1)
    return y[..., 0] if period == 1 else y


def conv1d_acc(x, w, *, stride=1, padding=(0, 0), dilation=1, groups=1, pad_mode="zero", period=1, pre_slope=1.0):
    """fp64 sum over (channel, tap) of w * lrelu(x) on the period view, rows padded by ``padding`` in ``pad_mode``.
    Returns (acc, per-element sum of the term magnitudes, the products' grid)."""
    B = x.shape[0]
    w = w.reshape(w.shape[0], w.shape[1], -1)
    xa = lrelu(x, pre_slope)
    xc = _pad(columns(xa.double(), period), padding[0], padding[1], pad_mode)
    kw = dict(stride=stride, dilation=dilation, groups=groups)
    acc = F.conv1d(xc, w.double(), **kw)
    bound = F.conv1d(xc.abs(), w.double().abs(), **kw)
    return uncolumns(acc, B, period), uncolumns(bound, B, period), grid(xa) * grid(w)


def conv1d(x, w, bias=None, *, stride=1, padding=(0, 0), dilation=1, groups=1, pad_mode="zero", period=1, pre_slope=1.0,
           post_act=None, post_slope=1.0, residual=None, out_scale=1.0, prev=None):
    """conv1d_fwd_kernel / small_cout / fewcout_long: y = [prev +] out_scale * (act(conv(lrelu(x)) + bias) + residual).
    x: (B, Cin, L) with L the valid length (t_valid) of the period view, or (B, Cin, rows, P).  post_act: None or
    "lrelu" (tanh is not exact: compare tanh of the None result within its ulp bound)."""
    if isinstance(padding, int):
        padding = (padding, padding)
    acc, bound, g = conv1d_acc(x, w, stride=stride, padding=padding, dilation=dilation, groups=groups, pad_mode=pad_mode,
                               period=period, pre_slope=pre_slope)
    return _epilogue(acc, bound, g, bias, post_act, post_slope, residual, out_scale, prev)


def virtual_weight(w, stride, groups=1):
    """(cin, cout / groups, K) -> the virtual conv's (cout * s, cin / groups, M) weight (convtr_weight_kernel):
    wv[co * s + ph][ci][m'] = w[g * cin_g + ci][co_l][ph + (M - 1 - m') * s], zero past K"""
    cin, cout_g, K = w.shape
    s, M = stride, -(-K // stride)
    cin_g = cin // groups
    wp = F.pad(w.double(), (0, M * s - K)).reshape(groups, cin_g, cout_g, M, s)  # [g][ci][co_l][m][ph], k = m s + ph
    wv = wp.flip(3).permute(0, 2, 4, 1, 3)  # [g][co_l][ph][ci][m']
    return wv.reshape(groups * cout_g * s, cin_g, M)


def conv_transpose1d(x, w, bias=None, *, stride, padding=0, output_padding=0, groups=1, period=1, pre_slope=1.0):
    """The FFMA conv-transpose as the kernel computes it: the virtual stride-1 conv (cout * s channels, ceil(K / s)
    taps, left pad M - 1) and the pixel-shuffle epilogue o = t * s + ph - padding, outputs outside [0, t_out) dropped.
    x: (B, cin, t_in[, P]), w: (cin, cout / groups, K).  Returns (y, Exactness)."""
    B, cin = x.shape[:2]
    t_in = x.shape[2]
    s, K = stride, w.shape[-1]
    M = -(-K // s)
    cout = w.shape[1] * groups
    t_out = (t_in - 1) * s - 2 * padding + K + output_padding
    tv = (t_out - 1 + padding) // s + 1
    wv = virtual_weight(w.reshape(cin, -1, K), s, groups)
    xf = x.reshape(B, cin, -1)
    acc, bound, g = conv1d_acc(xf, wv, padding=(M - 1, tv - t_in), groups=groups, period=period, pre_slope=pre_slope)

    def shuffle(v):
        v = v.reshape(B, cout, s, tv, period).permute(0, 1, 3, 2, 4).reshape(B, cout, tv * s, period)
        v = v[:, :, padding:padding + t_out]
        return v[..., 0] if period == 1 else v

    return _epilogue(shuffle(acc), shuffle(bound), g, bias, None, 1.0, None, 1.0, None)


def conv1d_wgrad(x, gy, kernel, *, stride=1, pad_left=0, dilation=1, groups=1, pad_mode="zero", period=1, x_slope=1.0,
                 g_slope=1.0, prev=None):
    """pwgb_conv1d_wgrad: dw[co, ci, k] (+)= sum_{b, t, p} gy'[b, co, t, p] x'[b, g cin_g + ci, t S + k D - pad, p] with
    gy' = lrelu(gy, g_slope), x' = lrelu(x, x_slope) on the (reflect-extended) period view, rows padded in ``pad_mode``.
    x: (B, Cin, L) flat, gy: (B, Cout, t_out[, P]).  Returns (dw (Cout, Cin / groups, K), Exactness)."""
    B, cin = x.shape[:2]
    cout = gy.shape[1]
    t_out = gy.shape[2]
    xa, ga = lrelu(x, x_slope), lrelu(gy, g_slope)
    xc = columns(xa.double(), period)
    gc = ga.double().reshape(B, cout, t_out, period).permute(0, 3, 1, 2).reshape(B * period, cout, t_out) if period > 1 \
        else ga.double().reshape(B, cout, t_out)
    need = (t_out - 1) * stride + (kernel - 1) * dilation + 1
    xc = _pad(xc, pad_left, need - pad_left - xc.shape[-1], pad_mode)
    cin_g, cout_g = cin // groups, cout // groups
    acc = torch.zeros(cout, cin_g, kernel, dtype=torch.float64)
    bound = torch.zeros_like(acc)
    for k in range(kernel):
        xk = xc[..., k * dilation:k * dilation + (t_out - 1) * stride + 1:stride]
        for g in range(groups):
            a, b = gc[:, g * cout_g:(g + 1) * cout_g], xk[:, g * cin_g:(g + 1) * cin_g]
            acc[g * cout_g:(g + 1) * cout_g, :, k] = torch.einsum("nct,ndt->cd", a, b)
            bound[g * cout_g:(g + 1) * cout_g, :, k] = torch.einsum("nct,ndt->cd", a.abs(), b.abs())
    return _epilogue(acc, bound, grid(xa) * grid(ga), None, None, 1.0, None, 1.0, prev)


def bias_grad(g, prev=None):
    """bias_grad_kernel / bias_grad_small_kernel: db[c] = [prev +] RN32(sum_{b, t} g[b, c, t]) (the sum in double)"""
    s = g.double().transpose(0, 1).reshape(g.shape[1], -1)
    db = s.sum(1).float()
    if prev is not None:
        db = prev.float() + db  # one fp32 addition, as the kernel
    return db, _double_exactness(s.abs().sum(1).max() if s.numel() else 0.0, grid(g))


def _nearest(x, s):
    return x.double().repeat_interleave(s, dim=-1)


def upsample_fir(x, fir, scale):
    """upsample_fir_kernel: y[r, o] = sum_k f[k] x[r, (o + k - s) / s] over 0 <= o + k - s < T s (nearest x s then the
    (2s+1)-tap FIR, zero padded).  The kernel pre-sums the taps per phase in fp32: their guard is part of the record."""
    s = scale
    f = fir.double().reshape(1, 1, -1)
    xr = _nearest(x, s)
    sh = xr.shape
    y = F.conv1d(xr.reshape(-1, 1, sh[-1]), f, padding=s).reshape(sh)
    bound = F.conv1d(xr.abs().reshape(-1, 1, sh[-1]), f.abs(), padding=s).reshape(sh)
    ex = Exactness(float(bound.max()), grid(x) * grid(fir)) & Exactness(float(fir.double().abs().sum()), grid(fir))
    return y.float(), ex


def upsample_fir_backward_x(gy, fir, scale):
    """upsample_fir_backward_x_kernel, the adjoint of upsample_fir in x: gy (..., T s) -> gx (..., T)"""
    s = scale
    f = fir.double().reshape(1, 1, -1)
    sh = gy.shape
    T = sh[-1] // s

    def adj(v, ff):
        return F.conv_transpose1d(v.reshape(-1, 1, sh[-1]), ff, padding=s).reshape(*sh[:-1], T, s).sum(-1)

    gx = adj(gy.double(), f)
    return gx.float(), Exactness(float(adj(gy.double().abs(), f.abs()).max()), grid(gy) * grid(fir))


def upsample_fir_backward_f(x, gy, scale):
    """the filter adjoint: df[k] = RN32(sum_{r, o} gy[r, o] x[r, (o + k - s) / s]).  The kernels sum in fp32 within a
    row (one thread's share), in double across threads and rows: the fp32 guard is per row, the double one total."""
    s = scale
    xr = F.pad(_nearest(x, s), (s, s))
    g = gy.double()
    Ts = g.shape[-1]
    df = torch.stack([(g * xr[..., k:k + Ts]).sum() for k in range(2 * s + 1)])
    row = (g.abs().sum(-1) * x.double().abs().amax(-1)).reshape(-1)
    gg = grid(x) * grid(gy)
    ex = Exactness(float(row.max()) if row.numel() else 0.0, gg) & _double_exactness(row.sum() * 3, gg)
    return df.float(), ex


def s2d(x, groups, stride, pad_left, rows_out, period=1, cgo=0):
    """s2d_forward_kernel: (B, C, rows[, P]) -> (B, groups * cgo, rows_out[, P]), channel (g, r, cl) = g cgo + r Cg + cl
    reads x[g Cg + cl, s u + r - pad]; channels >= s Cg of a group are zero"""
    B, Cc = x.shape[:2]
    P = period
    xv = x.reshape(B, groups, Cc // groups, -1, P)
    Cg, rows_in = xv.shape[2], xv.shape[3]
    cgo = cgo or Cg * stride
    y = torch.zeros(B, groups, cgo, rows_out, P)
    u = torch.arange(rows_out)
    for r in range(stride):
        row = stride * u + r - pad_left
        m = (row >= 0) & (row < rows_in)
        y[:, :, r * Cg:(r + 1) * Cg, u[m]] = xv[:, :, :, row[m]]
    y = y.reshape(B, groups * cgo, rows_out, P)
    return (y[..., 0] if P == 1 else y), Exactness(0.0, math.inf)


def s2d_backward(gy, x_shape, groups, stride, pad_left, period=1, cgo=0):
    """s2d_backward_kernel, the adjoint gather: gx[c, row] = gy[g cgo + r Cg + cl, u] with row + pad = u s + r"""
    B, Cc = x_shape[:2]
    P = period
    Cg = Cc // groups
    cgo = cgo or Cg * stride
    gv = gy.reshape(B, groups, cgo, -1, P)
    rows_out = gv.shape[3]
    rows_in = math.prod(x_shape[2:]) // P
    gx = torch.zeros(B, groups, Cg, rows_in, P)
    u = torch.arange(rows_out)
    for r in range(stride):
        row = stride * u + r - pad_left
        m = (row >= 0) & (row < rows_in)
        gx[:, :, :, row[m]] = gv[:, :, r * Cg:(r + 1) * Cg, u[m]]
    return gx.reshape(x_shape), Exactness(0.0, math.inf)


def pad1d(x, pad_left, pad_right, mode):
    """pad1d_forward_kernel: ReflectionPad1d / ReplicationPad1d"""
    return F.pad(x.double(), (pad_left, pad_right), mode=mode).float(), Exactness(0.0, math.inf)


def pad1d_backward(gxp, t, pad_left, pad_right, mode):
    """pad1d_backward_kernel, the adjoint of pad1d (fp64 autograd): gx[t] = sum of gxp at every position that copies t"""
    xx = torch.zeros(*gxp.shape[:-1], t, dtype=torch.float64, requires_grad=True)
    F.pad(xx, (pad_left, pad_right), mode=mode).backward(gxp.double())
    bx = torch.zeros_like(xx, requires_grad=True)
    F.pad(bx, (pad_left, pad_right), mode=mode).backward(gxp.double().abs())
    return xx.grad.float(), Exactness(float(bx.grad.max()) if bx.numel() else 0.0, grid(gxp))


def _pool_div(t_in, t_out, k, s, pad, include_pad):
    start = torch.arange(t_out) * s - pad
    if include_pad:
        return torch.minimum(start + k, torch.tensor(t_in + pad)) - start
    return torch.minimum(start + k, torch.tensor(t_in)) - torch.clamp(start, min=0)


def _pool_matrix(t_in, k, s, pad):
    """(t_out, t_in) 0/1 window membership"""
    t_out = (t_in + 2 * pad - k) // s + 1
    i = torch.arange(t_in)
    start = (torch.arange(t_out) * s - pad).unsqueeze(1)
    return ((i >= start) & (i < start + k)).double()


def avg_pool1d(x, k, s, pad=0, include_pad=True):
    """avg_pool1d_kernel: RN32(RN32(window sum) / div), div = the count_include_pad policy's divisor"""
    A = _pool_matrix(x.shape[-1], k, s, pad)
    sm = torch.einsum("...i,oi->...o", x.double(), A)
    div = _pool_div(x.shape[-1], A.shape[0], k, s, pad, include_pad).float()
    bound = torch.einsum("...i,oi->...o", x.double().abs(), A)
    return sm.float() / div, Exactness(float(bound.max()), grid(x))


def avg_pool1d_backward(gy, t_in, k, s, pad=0, include_pad=True):
    """avg_pool1d_backward_kernel: gx[i] = sum over windows o containing i of RN32(gy[o] / div(o)).  The guard checks
    that every quotient is exact (gradients that are multiples of 12 make it so for divisors 1 to 4)."""
    A = _pool_matrix(t_in, k, s, pad)
    div = _pool_div(t_in, A.shape[0], k, s, pad, include_pad).double()
    q = gy.double() / div
    gx = torch.einsum("...o,oi->...i", q, A)
    bound = torch.einsum("...o,oi->...i", q.abs(), A)
    ex = Exactness(float(bound.max()), grid(q))
    exact_q = torch.equal(q.float().double(), q)
    return gx.float(), ex if exact_q else Exactness(math.inf, 1.0)


def act_backward(mode, g, ref=None, slope=0.0, scale=1.0, prev=None):
    """act_backward_kernel: out = [prev +] (g * scale) * f'(ref); mode "lrelu" (ref > 0 ? 1 : slope), "tanh"
    (1 - ref * ref, each step in fp32) or "scale".  The guard checks every intermediate value for exactness."""
    v = g.double() * scale
    steps = [v]
    if mode == "lrelu":
        v = v * torch.where(ref > 0, torch.ones_like(v), torch.full_like(v, slope))
    elif mode == "tanh":
        r2 = ref.double() * ref.double()
        d = 1.0 - r2
        v = v * d
        steps += [r2, d]
    steps.append(v)
    if prev is not None:
        v = v + prev.double()
        steps.append(v)
    return v.float(), _values_exactness(*steps)


def axpby(a, x, b, y):
    """axpby_kernel: a * x + (b == 0 ? 0 : b * y); with b = 0 the old y (NaN included) is not read into the result"""
    ax = a * x.double()
    v = ax if b == 0 else ax + b * y.double()
    steps = [ax, v] + ([] if b == 0 else [b * y.double()])
    return v.float(), _values_exactness(*steps)


def scaled_sum(xs, a):
    """scaled_sum_kernel: a x_0 + a x_1 + ... (one fma per input, index order)"""
    terms = [a * x.double() for x in xs]
    v = sum(terms)
    bound = sum(t.abs() for t in terms)
    return v.float(), Exactness(float(bound.max()), min(grid(t) for t in terms))
