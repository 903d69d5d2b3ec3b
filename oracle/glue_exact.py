"""float64 references and per-element error bounds for the kernels that sit between the convolutions: the fused
optimizer (optim.cu), InstanceNorm1d and the TADE glue (tade.cu), the channel LayerNorm (symbol.cu), the WaveNet gate
(backward.cu) and the loss reductions (reduce.cu, backward.cu).

Two kinds of reference, as in oracle/ffma_exact.py:

* exact: on data with few mantissa bits and power-of-two scales every fp32 product and every partial sum of the kernel is
  exact, so its result is unique whatever the summation order and whether or not a multiply-add is contracted.  Each
  such function asserts that precondition (``require_exact`` / ``require_sum_exact``) and returns fp32 values that the
  kernel must reproduce bit for bit.
* bounded: where the arithmetic is inexact by nature (division, sqrtf, rsqrtf, expf, tanhf, __expf) the function
  returns the float64 value and, per element, a bound on |kernel - value| derived from the unit roundoff U = 2^-24, the
  documented errors of the CUDA math functions (CUDA C Programming Guide, "Mathematical Functions": sqrtf and division
  correctly rounded, rsqrtf 2 ulp, expf 2 ulp, tanhf 2 ulp, logf 1 ulp, __expf 2 + floor(1.173 |x|) ulp), the depth of
  the sums and the conditioning of the row.  One ulp is 2 U relative.  The derivations are first order; ``SLACK`` covers
  the second-order terms.

numpy float64 and Python numbers only; no CUDA, no torch arithmetic.  CPU only."""
import math

import numpy as np

U = 2.0 ** -24  # unit roundoff of fp32
SLACK = 1.25  # second-order terms of the first-order bounds below
TINY = 2.0 ** -126  # results below the smallest normal fp32 may be flushed or lose bits
F32 = np.float32


def f64(a):
    return np.asarray(a, dtype=np.float64)


def is_f32(v):
    v = f64(v)
    with np.errstate(over="ignore"):
        return bool(np.array_equal(v.astype(F32).astype(np.float64), v))


def require_exact(**vs):
    """every named float64 array holds values an fp32 operation produces without rounding"""
    for k, v in vs.items():
        assert is_f32(v), f"exactness precondition: {k} is not representable in fp32"


def lsb(v):
    """the smallest power of two of which every element of v is a multiple (inf for all zeros)"""
    v = np.abs(f64(v).reshape(-1))
    v = v[v != 0]
    if v.size == 0:
        return math.inf
    m, e = np.frexp(v)
    n = np.ldexp(m, 53).astype(np.int64)
    low = (n & -n).astype(np.float64)
    return float(np.ldexp(low, e - 53).min())


def require_sum_exact(abs_sums, terms, what, bits=24):
    """sums whose terms are multiples of g = lsb(terms) and whose absolute sums stay below 2^bits g are exact in any order"""
    g = lsb(terms)
    top = float(np.max(abs_sums)) if np.size(abs_sums) else 0.0
    assert top < math.ldexp(g, bits), f"exactness precondition: {what}: sum {top} reaches 2^{bits} x grid {g}"


def ratio(got, ref, bound):
    """worst |got - ref| / bound over the elements (inf where a non-finite value disagrees)"""
    got, ref, bound = f64(got), f64(ref), np.broadcast_to(f64(bound), np.shape(ref))
    if got.size == 0:
        return 0.0
    bad = ~np.isfinite(got)
    err = np.where(bad, np.inf, np.abs(np.where(bad, 0.0, got) - ref))
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.max(r))


# ------------------------------------------------------------------------------------------------ fused optimizer
CHUNK = 8192


def grad_norm(grads):
    """(float)sqrt(double sum of squares): the value mt_clip_coef_kernel writes when its fp32 chunk sums are exact"""
    total = 0.0
    for g in grads:
        total += float((f64(g) ** 2).sum())
    return F32(np.sqrt(np.float64(total)))


def clip(grads, max_norm, exact=False):
    """(norm, coef) as fp32 scalars: coef = min(1, max_norm / (norm + 1e-6f)) in fp32, 1 when max_norm <= 0.
    ``exact`` asserts that every 8192-element chunk's sum of squares is exact in fp32 (then norm is bit for bit)."""
    if exact:
        for g in grads:
            sq = f64(g).reshape(-1) ** 2
            require_exact(squares=sq)
            pad = (-sq.size) % CHUNK
            require_sum_exact(np.pad(sq, (0, pad)).reshape(-1, CHUNK).sum(1) if sq.size else 0.0, sq, "chunk sum of squares")
    norm = grad_norm(grads)
    c = F32(1.0)
    if max_norm is not None and max_norm > 0:
        c = F32(max_norm) / (norm + F32(1e-6))
        c = F32(1.0) if c > F32(1.0) else c
    return norm, c


def clipped_grad(g, coef):
    """g * coef as the kernel forms it: one fp32 multiply"""
    return (np.asarray(g, F32) * F32(coef)).astype(F32)


def radam_mode(t, betas):
    """(mode, step_size) of radam.py:65-79: mode 1 rectified (n_sma >= 5), mode 2 not"""
    b1, b2 = betas
    beta2_t = b2 ** t
    n_max = 2.0 / (1.0 - b2) - 1.0
    n_sma = n_max - 2.0 * t * beta2_t / (1.0 - beta2_t)
    if n_sma >= 5:
        return 1, math.sqrt((1 - beta2_t) * (n_sma - 4) / (n_max - 4) * (n_sma - 2) / n_sma * n_max / (n_max - 2)) / (1 - b1 ** t)
    return 2, 1.0 / (1 - b1 ** t)


def _r(x):
    return float(F32(x))  # a Python double as the kernel receives it


def optim_step(kind, p, g, m, v, t, lr, betas, eps, wd=0.0, coef=None, exact_state=False):
    """One step of Adam (``kind`` "adam": torch.optim.Adam, amsgrad=False) or RAdam ("radam": radam.py:27-99) in float64
    from the fp32 state (p, g, m, v) before the step; t is the step count after it.  The scalars are the ones the
    kernel receives (the Python doubles rounded to fp32, 1 - beta formed in fp32).  Returns a dict with p, m, v
    (float64) and bp, bm, bv, per-element bounds on the kernel's error:

      g' = g * coef is one fp32 multiply (reproduced exactly); with Adam weight decay g' = fma(wd, p, g'), U |g'|.
      m = b1 m + (1 - b1) g': two products and a sum (or one product and a fused multiply-add): 2 U (|b1 m| + |(1-b1) g'|).
      v = b2 v + ((1 - b2) g') g': three products and a sum: 3 U (b2 v + (1-b2) g'^2).
      update = c1 * (m / (sqrtf(v) * c2 + eps)): sqrtf and the division are correctly rounded, so one rounding each for
      sqrtf, * c2, + eps, /, * c1 (5 U, 5.5 with the half-weight of v's own rounding budget), plus the errors of m and v
      carried through; p - update rounds once more (U |p|).  RAdam's decay p -= (wd * lr) * p adds 2 U |wd lr p| + U |p|.

    ``exact_state`` asserts that m and v are exact in fp32 (every product and both sums), so they must match bit for bit."""
    p, g, m, v = f64(p), f64(g), f64(m), f64(v)
    b1, b2 = _r(betas[0]), _r(betas[1])
    omb1, omb2 = float(F32(1.0) - F32(betas[0])), float(F32(1.0) - F32(betas[1]))
    lr_, eps_, wd_ = _r(lr), _r(eps), _r(wd)
    if coef is not None:
        g = f64(clipped_grad(g, coef))
    eg = np.zeros_like(g)
    if kind == "adam":
        mode, c1, c2 = 0, _r(lr / (1.0 - betas[0] ** t)), _r(1.0 / math.sqrt(1.0 - betas[1] ** t))
        if wd != 0:
            g = g + wd_ * p
            eg = U * np.abs(g)
    else:
        mode, step_size = radam_mode(t, betas)
        c1, c2 = _r(step_size * lr), 1.0
    t1, t2 = b1 * m, omb1 * g
    m1 = t1 + t2
    s1, s2 = b2 * v, (omb2 * g) * g
    v1 = s1 + s2
    if exact_state:
        require_exact(b1_m=t1, omb1_g=t2, m=m1, b2_v=s1, omb2_g=omb2 * g, omb2_g_g=s2, v=v1)
    bm = 2.25 * U * (np.abs(t1) + np.abs(t2)) + omb1 * eg
    bv = 3.25 * U * (s1 + s2) + omb2 * 2.01 * np.abs(g) * eg
    p1 = p
    bp = np.zeros_like(p)
    if mode != 0 and wd != 0:
        p1 = p - (wd_ * lr_) * p
        bp = U * np.abs(p1) + 2 * U * np.abs(wd_ * lr_ * p)
    if mode == 2:
        upd = c1 * m1
        bu = U * np.abs(upd) + c1 * bm
    else:
        denom = np.sqrt(v1) * c2 + eps_
        upd = c1 * (m1 / denom)
        with np.errstate(divide="ignore", invalid="ignore"):
            rv = np.where(v1 > 0, 0.5 * bv / v1, 0.0)
        bu = np.abs(upd) * (5.5 * U + rv) + c1 * bm / denom
    p2 = p1 - upd
    bp = SLACK * (bp + bu + U * np.abs(p2))
    return dict(p=p2, m=m1, v=v1, bp=bp, bm=SLACK * bm, bv=SLACK * bv, mode=mode)


# ------------------------------------------------------------------------------------------------ TADE glue, exact
def lrelu(x, slope):
    x = f64(x)
    return np.where(x > 0, x, x * float(F32(slope)))


def leaky_relu_exact(x, slope):
    y = lrelu(x, slope)
    require_exact(leaky_relu=y)
    return y.astype(F32)


def upsample_nearest(x, scale):
    """y[..., o] = x[..., o / scale]"""
    return np.repeat(np.asarray(x), scale, axis=-1)


def upsample_nearest_backward_exact(gy, scale):
    """gx[..., i] = sum_j gy[..., i * scale + j]"""
    gy = f64(gy)
    g = gy.reshape(gy.shape[:-1] + (gy.shape[-1] // scale, scale))
    require_sum_exact(np.abs(g).sum(-1), gy, "upsample_nearest_backward")
    return g.sum(-1).astype(F32)


def tade_combine_exact(cg, xn, scale):
    """y[b, c, o] = cg[b, c, o] * xn[b, c, o / scale] + cg[b, C + c, o]"""
    cg, xn = f64(cg), f64(xn)
    C = cg.shape[1] // 2
    prod = cg[:, :C] * upsample_nearest(xn, scale)
    y = prod + cg[:, C:]
    require_exact(tade_combine_product=prod, tade_combine=y)
    return y.astype(F32)


def tade_combine_backward_exact(cg, xn, gy, scale):
    """(gcg, gxn): gcg[:, :C] = gy * up(xn), gcg[:, C:] = gy, gxn[i] = sum_j gy[i s + j] * cg[:, :C][i s + j]"""
    cg, xn, gy = f64(cg), f64(xn), f64(gy)
    C = cg.shape[1] // 2
    g1 = gy * upsample_nearest(xn, scale)
    terms = gy * cg[:, :C]
    require_exact(gcg=g1, gxn_terms=terms)
    grp = terms.reshape(terms.shape[:-1] + (terms.shape[-1] // scale, scale))
    require_sum_exact(np.abs(grp).sum(-1), terms, "tade_combine_backward gxn")
    return np.concatenate([g1, gy], 1).astype(F32), grp.sum(-1).astype(F32)


# ------------------------------------------------------------------------------------------------ InstanceNorm1d, bounded
def _in_depth(t):
    return -(-t // 256) + 13  # per-thread serial terms, 5 shuffle levels, 8 warp partials


def _instance_stats(x, eps, pre_slope):
    """float64 statistics of each row of x (rows, t) and the error budget of the kernel's own statistics.

    Sums: a thread adds ceil(t / 256) terms, the block tree 13 more: |sum error| <= depth U sum|terms|.
    mean: em = (depth + 1) U mean|a| (+ U mean|a| when the LeakyReLU product rounds, i.e. slope is not a power of two).
    variance, two-pass: a shift d of the mean moves sum((a - mean)^2) / t by d^2 only (the cross term sums to zero), so
      dvar = (depth + 4) U var + em^2 + 2 sqrt(var) ea + ea^2, ea the rms input rounding.
    rstd = rsqrtf(var + eps): 2 ulp = 4 U, one rounding each for / t and + eps: relative 0.5 dvar / (var + eps) + 6 U."""
    x = f64(x)
    t = x.shape[-1]
    a = lrelu(x, pre_slope)
    sl = float(F32(pre_slope))
    pow2 = sl == 0 or math.frexp(sl)[0] == 0.5
    ea_i = np.zeros_like(a) if pow2 else np.where(x > 0, 0.0, U * np.abs(a))
    d = _in_depth(t)
    mean = a.mean(-1, keepdims=True)
    em = (d + 1) * U * np.abs(a).mean(-1, keepdims=True) + ea_i.mean(-1, keepdims=True)
    c = a - mean
    var = (c * c).mean(-1, keepdims=True)
    ea = np.sqrt((ea_i ** 2).mean(-1, keepdims=True))
    dvar = (d + 4) * U * var + em ** 2 + 2 * np.sqrt(var) * ea + ea ** 2
    w = var + _r(eps)
    rstd = 1.0 / np.sqrt(w)
    r_rel = 0.5 * dvar / w + 6 * U
    return a, ea_i, mean, em, c, rstd, r_rel, d


def instance_norm(x, eps, pre_slope=1.0):
    """(y, bound) of InstanceNorm1d on rows of (rows, t): biased variance, eps inside the root, LeakyReLU first.
    y = (a - mean) * rstd:  |dy| <= rstd (em + ea_i) + |y| (r_rel + 2 U)  (the subtraction and the product round once each)."""
    a, ea_i, mean, em, c, rstd, r_rel, _ = _instance_stats(x, eps, pre_slope)
    y = c * rstd
    by = rstd * (em + ea_i) + np.abs(y) * (r_rel + 2 * U)
    return y, SLACK * by + TINY


def instance_norm_backward(x, gy, eps, pre_slope=1.0):
    """(gx, bound): ga = rstd (gy - m1 - yh m2), m1 = mean(gy), m2 = mean(gy yh), gx = ga * lrelu'(x).
    e1 = (depth + 1) U mean|gy|;  e2 = (depth + 2) U mean|gy yh| + mean(|gy| dyh);  the bracket rounds three times:
    |dga| <= rstd (e1 + |yh| e2 + dyh |m2| + 3 U (|gy| + |m1| + |yh m2|)) + |ga| (r_rel + 2 U)."""
    a, ea_i, mean, em, c, rstd, r_rel, d = _instance_stats(x, eps, pre_slope)
    gy = f64(gy)
    yh = c * rstd
    dyh = rstd * (em + ea_i) + np.abs(yh) * (r_rel + 2 * U)
    m1 = gy.mean(-1, keepdims=True)
    m2 = (gy * yh).mean(-1, keepdims=True)
    e1 = (d + 1) * U * np.abs(gy).mean(-1, keepdims=True)
    e2 = (d + 2) * U * np.abs(gy * yh).mean(-1, keepdims=True) + (np.abs(gy) * dyh).mean(-1, keepdims=True)
    ga = rstd * (gy - m1 - yh * m2)
    bga = rstd * (e1 + np.abs(yh) * e2 + dyh * np.abs(m2) + 3 * U * (np.abs(gy) + np.abs(m1) + np.abs(yh * m2))) + np.abs(ga) * (r_rel + 2 * U)
    sl = np.where(f64(x) > 0, 1.0, float(F32(pre_slope)))
    return ga * sl, SLACK * (bga * np.abs(sl) + U * np.abs(ga * sl)) + TINY


# ------------------------------------------------------------------------------------------------ TADE gate, bounded
def _softmax_gate(xa):
    """(g, relative bound) of the kernel's softmax over axis 1.  expf is 2 ulp (4 U) and its argument a - max rounds
    once (U |a - max| absolute, the same relative to the exponential); the denominator adds C positive terms (C U),
    carries the weighted argument errors of its terms, is inverted (U) and multiplied (U)."""
    xa = f64(xa)
    C = xa.shape[1]
    z = xa - xa.max(1, keepdims=True)
    e = np.exp(z)
    s = e.sum(1, keepdims=True)
    g = e / s
    rel = (4 + np.abs(z)) * U + (4 + C) * U + U * (g * np.abs(z)).sum(1, keepdims=True) + 2 * U
    return g, rel


def _sigmoid_gate(xa):
    """1 / (1 + expf(-a)): expf 4 U, the sum and the division one rounding each: 6 U relative"""
    xa = f64(xa)
    with np.errstate(over="ignore"):
        g = 1.0 / (1.0 + np.exp(-xa))
    return g, np.full_like(g, 6 * U)


def tade_gate(x, residual=None, scale=1, softmax=True):
    """(y, bound): y[b, c, t] = gate(xa)[b, c, t] * tanh(xb[b, c, t]) + residual[b, c, t / scale]; tanhf 2 ulp (4 U),
    the product U, the residual add U |y|."""
    x = f64(x)
    C = x.shape[1] // 2
    g, rel = (_softmax_gate if softmax else _sigmoid_gate)(x[:, :C])
    v = g * np.tanh(x[:, C:])
    by = np.abs(v) * (rel + 5 * U)
    y = v
    if residual is not None:
        y = v + upsample_nearest(f64(residual), scale)
        by = by + U * np.abs(y)
    return y, SLACK * by + TINY


def tade_gate_backward(x, gy, softmax=True):
    """(gx, bound), gx = [gxa | gxb]: u = gy tanh(xb);  softmax: gxa = g (u - dot), dot = sum_c g u;  sigmoid:
    gxa = u g (1 - g);  gxb = gy g (1 - tanh^2).  1 - tanh^2 and 1 - g cancel, so their error is absolute:
    d(1 - th^2) <= 9 U th^2 + U, d(1 - g) <= rel g + U."""
    x, gy = f64(x), f64(gy)
    C = x.shape[1] // 2
    g, rel = (_softmax_gate if softmax else _sigmoid_gate)(x[:, :C])
    th = np.tanh(x[:, C:])
    u = gy * th
    eu = 5 * U * np.abs(u)
    if softmax:
        dot = (g * u).sum(1, keepdims=True)
        edot = (np.abs(g * u) * (rel + 6 * U + C * U)).sum(1, keepdims=True)
        gxa = g * (u - dot)
        ba = np.abs(g) * (eu + edot + U * np.abs(u - dot)) + np.abs(gxa) * (rel + U)
    else:
        gxa = u * g * (1 - g)
        ba = np.abs(u * g) * (rel * g + U) + np.abs(gxa) * (rel + 8 * U)
    gxb = gy * g * (1 - th * th)
    bb = np.abs(gy * g) * (9 * U * th * th + U) + np.abs(gxb) * (rel + 3 * U)
    return np.concatenate([gxa, gxb], 1), SLACK * np.concatenate([ba, bb], 1) + TINY


# ------------------------------------------------------------------------------------------------ channel LayerNorm
def _ln_depth(C):
    return -(-C // 8) + 8  # each of 8 warps adds ceil(C / 8) terms, one thread adds the 8 partials


def channel_layernorm(x, gamma, beta, eps):
    """LayerNorm over axis 1 of (B, C, T).  Returns y, mean, rstd (float64) and by, bmean, brstd.
    mean: em = (depth + 1) U mean|x|.  Variance, two-pass: dvar = (depth + 4) U var + em^2.  rstd = 1 / sqrtf(var + eps),
    both correctly rounded, / C and + eps one rounding each: relative 0.5 dvar / (var + eps) + 4 U.
    y = ((x - mean) rstd) gamma + beta: |dy| <= |rstd gamma| em + |xhat gamma| (r_rel + 3 U) + U |y|."""
    x, gamma, beta = f64(x), f64(gamma).reshape(1, -1, 1), f64(beta).reshape(1, -1, 1)
    d = _ln_depth(x.shape[1])
    mean = x.mean(1, keepdims=True)
    em = (d + 1) * U * np.abs(x).mean(1, keepdims=True)
    c = x - mean
    var = (c * c).mean(1, keepdims=True)
    w = var + _r(eps)
    dvar = (d + 4) * U * var + em ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        rstd = 1.0 / np.sqrt(w)
        r_rel = np.where(w > 0, 0.5 * dvar / w, 0.0) + 4 * U
    xg = c * rstd * gamma
    y = xg + beta
    by = np.abs(rstd * gamma) * em + np.abs(xg) * (r_rel + 3 * U) + U * np.abs(y)
    return dict(y=y, mean=mean[:, 0], rstd=rstd[:, 0], by=SLACK * by + TINY, bmean=SLACK * em[:, 0] + TINY,
                brstd=SLACK * (rstd * r_rel)[:, 0] + TINY)


def channel_layernorm_backward(x, gy, gamma, mean, rstd):
    """Backward from the saved fp32 statistics (inputs, so they carry no error): xhat = (x - mean) rstd (2 U),
    dx = rstd (gy gamma - m1 - xhat m2), m1 = mean_c(gy gamma), m2 = mean_c(gy gamma xhat);
    dgamma = sum_{b,t} gy xhat, dbeta = sum_{b,t} gy: a 5-level warp tree over 32 frames, then B ceil(T / 32) block
    partials added in order: |d sum| <= (5 + B ceil(T / 32) + 3) U sum|terms|, a bound that grows with B * T.
    Returns dx, dgamma, dbeta and bdx, bdgamma, bdbeta."""
    x, gy, gamma = f64(x), f64(gy), f64(gamma).reshape(1, -1, 1)
    mean, rstd = f64(mean)[:, None], f64(rstd)[:, None]
    B, C, T = x.shape
    d = _ln_depth(C)
    xh = (x - mean) * rstd
    gg = gy * gamma
    m1 = gg.mean(1, keepdims=True)
    m2 = (gg * xh).mean(1, keepdims=True)
    e1 = (d + 2) * U * np.abs(gg).mean(1, keepdims=True)
    e2 = (d + 5) * U * np.abs(gg * xh).mean(1, keepdims=True)
    dx = rstd * (gg - m1 - xh * m2)
    bdx = np.abs(rstd) * (e1 + np.abs(xh) * e2 + 3 * U * np.abs(xh * m2) + 3 * U * (np.abs(gg) + np.abs(m1) + np.abs(xh * m2))) + U * np.abs(dx)
    depth = 5 + B * (-(-T // 32)) + 3
    tg = gy * xh
    return dict(dx=dx, dgamma=tg.sum((0, 2)), dbeta=gy.sum((0, 2)), bdx=SLACK * bdx + TINY,
                bdgamma=SLACK * depth * U * np.abs(tg).sum((0, 2)) + TINY, bdbeta=SLACK * depth * U * np.abs(gy).sum((0, 2)) + TINY)


def channel_layernorm_param_grads_exact(x, gy, mean, rstd):
    """dgamma, dbeta bit for bit: with mean, rstd and x chosen so that xhat = (x - mean) rstd, the products gy xhat and
    the sums over (b, t) are all exact"""
    x, gy = f64(x), f64(gy)
    xh = (x - f64(mean)[:, None]) * f64(rstd)[:, None]
    tg = gy * xh
    require_exact(xhat=xh, gy_xhat=tg)
    require_sum_exact(np.abs(tg).sum((0, 2)), tg, "dgamma")
    require_sum_exact(np.abs(gy).sum((0, 2)), gy, "dbeta")
    return tg.sum((0, 2)).astype(F32), gy.sum((0, 2)).astype(F32)


# ------------------------------------------------------------------------------------------------ WaveNet gate
def _fast_sigmoid(s):
    """(sg, relative bound) of 1 / (1 + __expf(-s)): __expf is 2 + floor(1.173 |s|) ulp, i.e. (4 + 2.346 |s|) U on
    e = exp(-s); d sg / sg = (1 - sg) de / e; the sum and the division round once each."""
    s = f64(s)
    with np.errstate(over="ignore"):
        sg = 1.0 / (1.0 + np.exp(-s))
    return sg, (1 - sg) * (4 + 2.346 * np.abs(s)) * U + 2 * U


def gate(g):
    """(z, bound): z[b, h, t] = tanh(g[b, h, t]) * sigmoid(g[b, H + h, t]); tanhf 4 U, the product U.  Below the
    smallest normal number (s < -87) the kernel's sigmoid may flush to zero: TINY absolute."""
    g = f64(g)
    H = g.shape[1] // 2
    ta = np.tanh(g[:, :H])
    sg, rel = _fast_sigmoid(g[:, H:])
    z = ta * sg
    return z, SLACK * np.abs(z) * (rel + 5 * U) + TINY


def gate_backward(g, gz):
    """(gg, bound), gg = [da | ds]: da = go sg (1 - ta^2), ds = go ta sg (1 - sg).  Both brackets cancel near saturation,
    so their errors are absolute, in units of |go|: d(1 - ta^2) <= 9 U ta^2 + U, d(1 - sg) <= rel sg + U."""
    g, go = f64(g), f64(gz)
    H = g.shape[1] // 2
    ta = np.tanh(g[:, :H])
    sg, rel = _fast_sigmoid(g[:, H:])
    da = go * sg * (1 - ta * ta)
    ds = go * ta * sg * (1 - sg)
    ba = np.abs(go * sg) * (9 * U * ta * ta + U) + np.abs(da) * (rel + 3 * U)
    bs = np.abs(go * ta * sg) * (rel * sg + U) + np.abs(ds) * (rel + 8 * U)
    return np.concatenate([da, ds], 1), SLACK * np.concatenate([ba, bs], 1) + TINY


# ------------------------------------------------------------------------------------------------ loss reductions
REDUCE_MODES = {"mse_const": 0, "l1": 1, "hinge": 2, "linear": 3, "mse": 4}


def reduce_terms(mode, x, y=None, c=0.0, s=1.0):
    """float64 terms of pwgb_reduce_mean_forward and the intermediate values whose exactness the exact case needs"""
    x = f64(x).reshape(-1)
    c, s = _r(c), _r(s)
    if mode == "mse_const":
        e = x - c
        return e * e, (e,)
    if mode == "l1":
        return np.abs(x - f64(y).reshape(-1)), ()
    if mode == "mse":
        e = x - f64(y).reshape(-1)
        return e * e, (e,)
    if mode == "hinge":
        return np.maximum(0.0, c - s * x), (s * x,)
    return s * x, ()


def reduce_blocks(n, ws_floats=1024):
    """the partial kernel's grid: min(ceil(n / 2048), ws_floats, 1024) blocks of 256 threads, grid-stride"""
    return max(1, min(-(-n // 2048), ws_floats, 1024))


def reduce_mean_exact(mode, x, y=None, c=0.0, s=1.0, weight=1.0, prev=None, ws_floats=1024):
    """out = (prev if accumulating) + (float)(double sum * ((double)weight / n)) on data whose terms and whose per-block
    fp32 partial sums are exact (asserted per block of the launch geometry; the final sum is carried in double)."""
    terms, mids = reduce_terms(mode, x, y, c, s)
    require_exact(terms=terms, **{f"mid{i}": v for i, v in enumerate(mids)})
    n = terms.size
    nb = reduce_blocks(n, ws_floats)
    a = np.abs(terms)
    pad = (-n) % (nb * 256)
    require_sum_exact(np.pad(a, (0, pad)).reshape(-1, nb, 256).sum((0, 2)), terms, "reduce_mean block partial")
    require_sum_exact(a.sum(), terms, "reduce_mean total", bits=52)
    val = F32(float(terms.sum()) * (float(F32(weight)) / float(n)))
    return val if prev is None else F32(prev) + val


def reduce_mean_backward_exact(mode, x, y=None, c=0.0, s=1.0, weight=1.0, gout=1.0, prev=None):
    """gx = (prev if accumulating) + go * f'(x[, y]) with go = gout * weight / (float)n formed in fp32; go * f' and the
    sum with prev must be exact (weight / n a power of two, small-integer data)."""
    x = f64(x).reshape(-1)
    n = x.size
    go = float(F32(F32(gout) * F32(weight)) / F32(n))
    c_, s_ = _r(c), _r(s)
    if mode == "mse_const":
        d = 2.0 * (x - c_)
    elif mode == "l1":
        d = np.sign(x - f64(y).reshape(-1))
    elif mode == "hinge":
        d = np.where(c_ - s_ * x > 0, -s_, 0.0)
    elif mode == "mse":
        d = 2.0 * (x - f64(y).reshape(-1))
    else:
        d = np.full_like(x, s_)
    t = go * d
    out = t if prev is None else f64(prev).reshape(-1) + t
    require_exact(d=d, go_d=t, gx=out)
    return out.astype(F32)


# ------------------------------------------------------------------------------------------------ duration loss
def duration_loss(x, ds, offset):
    """(loss, bound, gx per unit gout, bound): mean((x - log(ds + offset))^2), sum carried in double; logf 1 ulp (2 U),
    (float)ds + offset and the subtraction one rounding each: |dr| <= 3 U |log| + U |r|, d(r^2) <= 2 |r| dr + U r^2."""
    x, ds = f64(x).reshape(-1), f64(ds).reshape(-1)
    lg = np.log(ds + _r(offset))
    r = x - lg
    dr = 3 * U * np.abs(lg) + U * np.abs(r) + U  # + U: the argument's rounding, d log = d arg / arg <= U
    loss = float((r * r).mean())
    bl = float((2 * np.abs(r) * dr + U * r * r).mean()) + U * loss
    n = x.size
    gx = 2.0 / n * r
    return loss, SLACK * bl + TINY, gx, SLACK * (2.0 / n * dr + 3 * U * np.abs(gx)) + TINY


# ------------------------------------------------------------------------------------------------ symbol embedding
def symbol_embed_backward_exact(gy, idx, num_embs):
    """d_table[k, c] = sum over the positions (b, s) with idx[b, s] == k of gy[b, c, s] (no durations), exact sums"""
    gy = f64(gy)
    B, C, S = gy.shape
    idx = np.asarray(idx).reshape(B, S)
    out = np.zeros((num_embs, C))
    ab = np.zeros((num_embs, C))
    flat = gy.transpose(0, 2, 1).reshape(B * S, C)
    np.add.at(out, idx.reshape(-1), flat)
    np.add.at(ab, idx.reshape(-1), np.abs(flat))
    require_sum_exact(ab, gy, "symbol_embed_backward")
    return out.astype(F32)


# ------------------------------------------------------------------------------------------------ test data
def ints(rng, shape, k, scale=1.0):
    """fp32 values n * scale with integer |n| <= k: few mantissa bits, every element drawn independently"""
    return (rng.integers(-k, k + 1, size=shape).astype(np.float64) * scale).astype(F32)


def instance_rows(kind, rows, t, seed):
    """rows for InstanceNorm1d: "plain" mean 0.7 std 3; "offset" mean 100 std 1e-2 (a one-pass variance loses it);
    "const" a constant row whose sums are exact (output exactly 0); "tiny" std 1e-4, so eps = 1e-5 dominates the variance"""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((rows, t))
    if kind == "plain":
        x = 0.7 + 3.0 * z
    elif kind == "offset":
        x = 100.0 + 1e-2 * z
    elif kind == "const":
        x = np.full((rows, t), 2.5)
    else:
        x = 1e-4 * z
    return x.astype(F32)


# (rows, t, pre_slope, eps, kind)
INSTANCE_CASES = [
    (3, 1, 1.0, 1e-5, "plain"), (3, 2, 1.0, 1e-5, "plain"), (5, 2, 0.2, 1e-5, "plain"), (4, 255, 0.2, 1e-5, "plain"),
    (4, 256, 1.0, 1e-5, "plain"), (4, 257, 0.2, 1e-5, "plain"), (6, 1000, 1.0, 1e-5, "plain"), (3, 22528, 0.2, 1e-5, "plain"),
    (4, 1000, 1.0, 1e-5, "offset"), (2, 22528, 1.0, 1e-5, "offset"), (4, 257, 0.2, 1e-5, "offset"), (3, 1000, 1.0, 1e-5, "const"),
    (3, 257, 0.2, 1e-5, "tiny"), (4, 1000, 1.0, 1e-5, "tiny"), (4, 31, 1.0, 0.0, "plain"),
]


def gate_logits(kind, B, C, T, seed):
    """(B, 2C, T) inputs of tade_gate: "unit" N(0, 1); "spread" gate logits uniform over +-80 around a per-column offset of
    -60, 0 or 60 (without the max subtraction expf overflows); "one" the same with tanh saturated at 1; "sat" gate inputs at
    +-100 and tanh inputs at +-20 (saturated: tanhf = +-1 exactly)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((B, 2 * C, T))
    if kind == "spread":
        x[:, :C] = rng.uniform(-80, 80, (B, C, T)) + rng.choice([-60.0, 0.0, 60.0], (B, 1, T))
        x[:, C:] *= 3
    elif kind == "sat":
        x[:, :C] = rng.choice([-100.0, -30.0, 0.0, 30.0, 100.0], (B, C, T))
        x[:, C:] = rng.choice([-20.0, 20.0], (B, C, T))
    elif kind == "one":
        x[:, :C] = rng.uniform(-80, 80, (B, C, T))
        x[:, C:] = 20.0
    return x.astype(F32)


# (B, C, T, scale, softmax, residual, kind)
TADE_GATE_CASES = [
    (2, 1, 37, 1, True, False, "unit"), (2, 2, 64, 2, True, True, "spread"), (1, 64, 96, 4, True, True, "spread"),
    (2, 64, 33, 1, True, False, "one"), (2, 1, 40, 1, False, False, "sat"), (2, 2, 60, 3, False, True, "sat"),
    (1, 64, 128, 8, False, True, "unit"), (3, 5, 50, 5, True, True, "sat"), (1, 2, 540672 + 2048 + 5, 1, True, False, "spread"),
    (1, 1, 540672 + 2 * 2048, 2, False, True, "sat"),
]

# (B, C, T, eps, kind): "plain" N(0.3, 2); "offset" a common offset of 50 on std 0.05; "gamma0" gamma all zero
LAYERNORM_CASES = [
    (1, 1, 1, 1e-5, "plain"), (3, 7, 31, 1e-12, "plain"), (1, 8, 32, 1e-5, "plain"), (3, 9, 33, 1e-12, "plain"),
    (1, 64, 1000, 1e-12, "plain"), (3, 384, 33, 1e-5, "plain"), (1, 1000, 31, 1e-12, "plain"), (1, 7, 5000, 1e-5, "plain"),
    (3, 64, 1000, 1e-12, "offset"), (1, 384, 32, 1e-5, "offset"), (3, 9, 1, 1e-12, "plain"), (1, 64, 33, 1e-12, "gamma0"),
    (3, 8, 5000, 1e-12, "plain"),
]


def layernorm_data(B, C, T, kind, seed):
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((B, C, T))
    x = 50.0 + 0.05 * z if kind == "offset" else 0.3 + 2.0 * z
    gamma = np.zeros(C) if kind == "gamma0" else 1.0 + 0.5 * rng.standard_normal(C)
    beta = 0.3 * rng.standard_normal(C)
    gy = rng.standard_normal((B, C, T))
    return x.astype(F32), gamma.astype(F32), beta.astype(F32), gy.astype(F32)


def wavenet_gate_inputs(B, H, T, seed):
    """(B, 2H, T) uniform over +-30 with +-88, +-200, 0 and +-20 planted at the start of the first rows"""
    rng = np.random.default_rng(seed)
    g = rng.uniform(-30, 30, (B, 2 * H, T))
    sp = np.array([0.0, 88.0, -88.0, 200.0, -200.0, 20.0, -20.0, 87.0, -87.0, 103.0, -103.0])
    k = min(T, sp.size)
    g[0, 0, :k] = sp[:k]
    g[0, H, :k] = sp[:k][::-1]
    g[-1, -1, -k:] = sp[:k]
    return g.astype(F32)


REDUCE_SIZES = [1, 255, 256, 257, 2047, 2048, 2049, 2097152, 2097153, 5000001]


def reduce_data(mode, n, seed, coarse=False):
    """(x, y, c, s): small integers / 4, every term exact; hinge inputs land exactly on c - s x == 0 and L1 pairs on
    x == y about one time in nine.  ``coarse`` draws from {-1, 0, 1}: a grid clamped to a few blocks adds millions of
    terms per block, which stays exact only on a coarser grid"""
    rng = np.random.default_rng(seed)
    k, sc = (1, 1.0) if coarse else (4, 0.25)
    x = ints(rng, n, k, sc)
    y = ints(rng, n, k, sc) if mode in ("l1", "mse") else None
    c, s = {"mse_const": (1.0, 1.0), "l1": (0.0, 1.0), "hinge": (1.0, -1.0), "linear": (0.0, -1.0), "mse": (0.0, 1.0)}[mode]
    return x, y, c, s


OPTIM_EDGE_SIZES = [1, 2, 255, 256, 257, 8191, 8192, 8193, 16384, 3 * 8192 + 5]


def optim_big_sizes(count=320, seed=5):
    """sizes of a model with several hundred tensors: biases and small kernels, tensors around the chunk edges, a few large"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(count):
        k = i % 4
        if k == 0:
            out.append(int(rng.integers(1, 600)))
        elif k == 1:
            out.append(int(8192 * rng.integers(1, 4) + rng.integers(-2, 3)))
        elif k == 2:
            out.append(int(rng.integers(600, 20000)))
        else:
            out.append(int(rng.integers(1, 40)) * 512)
    return out


def optim_exact_tensors(sizes, seed, step):
    """gradients k / 64 with |k| <= 8, independent per tensor and step"""
    return [ints(np.random.default_rng([seed, step, i]), n, 8, 2.0 ** -6) for i, n in enumerate(sizes)]


def optim_random_tensors(sizes, seed, step, scale=1.0):
    return [(scale * np.random.default_rng([seed, step, i]).standard_normal(n)).astype(F32) for i, n in enumerate(sizes)]
