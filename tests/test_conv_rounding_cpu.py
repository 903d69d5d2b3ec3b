"""The rounding oracle of oracle/bf16x3.py ("rounding on fp32") checked on the CPU, over the tables that
tests/test_gpu_conv_rounding.py runs:

- the one-hot probes are exact: every output element receives at most one non-zero pair, and hi + lo is exact in fp32;
- the bound is honest: a plain fp32 evaluation in another order (torch float32 convs of the three bf16x3 terms) and the
  float64 conv of the same terms both stay inside it;
- the tests have teeth: each plausible kernel mistake, applied to the emulation, changes a readback somewhere (or
  leaves the bound), so the GPU comparison would fail;
- ``check_coverage`` of the GPU tables holds."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_gpu_conv_rounding as G
from oracle import bf16x3 as E

f32 = np.float32


def test_check_coverage():
    G.check_coverage()


def test_fp32_values_cover_every_class():
    x = E.fp32_values((200000,), 1, special=True)
    u = x.view(torch.int32).numpy().view(np.uint32)
    mag = u & 0x7FFFFFFF
    fin = torch.isfinite(x).numpy()
    assert (mag == 0).any() and ((mag > 0) & (mag < 0x00800000)).any(), "zeros and subnormals"
    assert ((mag & 0xFFFF) == 0x8000).any() and (((mag >> 16) & 1) == 0)[(mag & 0xFFFF) == 0x8000].any()
    assert (((mag >> 16) & 1) == 1)[(mag & 0xFFFF) == 0x8000].any(), "ties of both parities"
    assert ((mag >= E.BF16_INF_FROM) & fin).any() and (mag == 0x7F800000).any() and torch.isnan(x).any()
    assert (u >> 31).any() and not (u >> 31).all()
    hi, lo = E.split(x[torch.isfinite(x)])
    r = (x[torch.isfinite(x)].double() - hi.double())
    assert bool(((r - lo.double()).abs() == (lo.double().abs() * 2.0 ** -8)).any()), "lo ties"
    y = E.fp32_values((200000,), 1)
    assert bool(torch.isfinite(y).all()) and int((y.view(torch.int32) & 0x7FFFFFFF).max()) < E.BF16_INF_FROM


def test_split_is_round_to_nearest_even():
    x = E.from_bits(np.array([0x3F808000, 0x3F818000, 0x3F807FFF, 0x7F7F7FFF, 0x7F7F8000, 0x00000001, 0x80008000],
                             dtype=np.uint32))
    hi, lo = E.split(x)
    assert hi.view(torch.int32).tolist()[:3] == [0x3F800000, 0x3F820000, 0x3F800000]  # ties to even, below the tie
    assert math.isfinite(hi[3]) and hi[4] == math.inf and lo[4] == -math.inf
    assert hi[5] == 0 and lo[5] == 0  # 2^-149 is below bf16's smallest subnormal: both parts round to zero
    # below bf16's subnormal spacing (2^-133) a tie rounds to even twice: a subnormal fp32 may lose its low bits
    assert float(hi[6] + lo[6]) == 0.0 and float(x[6]) != 0.0


# ---------------------------------------------------------------------------------------------------- exactness
def _cases():
    for n in G.CONV:
        for p in G.PROBES:
            yield "conv", n, p
    for n in G.PAIR:
        for p in G.PAIR_PROBES:
            yield "pair", n, p
    for n in G.CONVTR:
        for p in G.PROBES:
            yield "convtr", n, p
    for n in G.STRIDED:
        for p in G.PROBES:
            yield "strided", n, p
    for n in G.WGRAD:
        for p in G.WGRAD_PROBES:
            yield "wgrad", n, p


def _exact_in_fp32(acc, what):
    fin = torch.isfinite(acc)
    assert torch.equal(acc[fin].float().double(), acc[fin]), f"{what}: an accumulator is not exact in fp32"


@pytest.mark.parametrize("kind,name,probe", list(_cases()))
def test_readback_cases_are_one_hot(kind, name, probe):
    """builds every launch of every GPU readback case (each asserts pair_count <= 1), checks that its finite
    accumulators are exact in fp32, and that the launches of a probe together read every input channel (of both
    sources, for the two-source conv-transpose)"""
    reads = set()
    if kind == "conv":
        n = G.CONV[name][1]
        for off in G.conv_offsets(name, probe):
            d, kw, ref, r = G.conv_case(name, probe, off)
            reads |= r
            _exact_in_fp32(E.conv1d_acc(d["x"], d["w"], **{k: kw[k] for k in ("padding", "dilation", "groups", "pad_mode",
                                                                               "pre_slope")})[0], name)
    elif kind == "pair":
        Cc, k, dil, _ = G.PAIR[name]
        n = Cc
        for off in G.pair_offsets(name, probe):
            d, ref, r = G.pair_case(name, probe, off)
            reads |= r
            _exact_in_fp32(E.conv1d_acc(d["x"], d["w1"], padding=((k - 1) // 2 * dil,) * 2, dilation=dil,
                                        pre_slope=0.1)[0], name)
    elif kind == "convtr":
        n = G.CONVTR[name][1] + G.CONVTR[name][2]
        for off in G.convtr_offsets(G.CONVTR[name], probe):
            x, w, b, kw, ref, r = G.convtr_case(name, probe, off)
            reads |= r
            _exact_in_fp32(E.conv_transpose1d_acc(x, w, pre_slope=0.1, **kw)[0], name)
        if G.CONVTR[name][2]:
            assert max(reads) >= G.CONVTR[name][1], f"{name}: the second source is never read"
    elif kind == "strided":
        cin, cout, K, s, groups, pad, rows, P, B = G.STRIDED[name][:9]
        n = cin
        for off in G.strided_offsets(name, probe):
            x, w, b, ref, r = G.strided_case(name, probe, off)
            reads |= r
            xc = x.view(B, cin, rows, P).permute(0, 3, 1, 2).reshape(B * P, cin, rows)
            _exact_in_fp32(E.conv1d_acc(xc, w, stride=s, padding=(pad, pad), groups=groups)[0], name)
    else:
        B, cin, cout, k, dil, pad, T, groups, xs, gs, _ = G.WGRAD[name]
        x, gy, ref = G.wgrad_case(name, probe)
        _exact_in_fp32(E.conv1d_wgrad_acc(x, gy, k, pad_left=pad, dilation=dil, groups=groups, x_slope=xs, g_slope=gs)[0],
                       name)
        n, reads = cin, G._channels(x) if probe == "gy" else set(range(cin))
    assert reads == set(range(n)), f"{name}/{probe}: {len(reads)} of {n} input channels read"
    assert ref.numel() > 0


# ---------------------------------------------------------------------------------------------------- honest bound
def _f32_terms(x, w, kw):
    """a plain fp32 evaluation of the bf16x3 conv in another order: three float32 convs, summed in float32"""
    xh, xl = E.split(x)
    wh, wl = E.split(w)
    return (F.conv1d(xh, wh, **kw) + F.conv1d(xl, wh, **kw)) + F.conv1d(xh, wl, **kw)


@pytest.mark.parametrize("cin,K,d,post,res,scale", [(64, 7, 3, None, True, G.THIRD), (128, 3, 1, "lrelu", False, 1.0),
                                                    (32, 11, 5, "tanh", False, 1.0)])
def test_bound_holds_for_fp32_and_float64(cin, K, d, post, res, scale):
    g = torch.Generator().manual_seed(cin + K)
    x = torch.randn(2, cin, 600, generator=g)
    w = torch.randn(cin, cin, K, generator=g) / math.sqrt(cin * K)
    b = torch.randn(cin, generator=g) * 0.1
    r = torch.randn(2, cin, 600, generator=g) if res else None
    prev = torch.randn(2, cin, 600, generator=g) if res else None
    p = (K - 1) // 2 * d
    acc, mag, _ = E.conv1d_acc(x, w, padding=(p, p), dilation=d, pre_slope=0.1)
    ref, beta = E.epilogue_f32(acc, b, post, 0.2, r, scale, prev, err=E.accumulation_bound(mag, 3 * cin * K, E.U_TC))
    a = F.pad(E.lrelu(x, 0.1), (p, p))
    y32 = E.epilogue_f32(_f32_terms(a, w, dict(dilation=d)), b, post, 0.2, r, scale, prev)
    y64 = E.epilogue_f32(F.conv1d(E.split(a)[0].double(), E.split(w)[0].double(), dilation=d) +
                         F.conv1d(E.split(a)[1].double(), E.split(w)[0].double(), dilation=d) +
                         F.conv1d(E.split(a)[0].double(), E.split(w)[1].double(), dilation=d), b, post, 0.2, r, scale, prev)
    for y in (y32, y64):
        ratio = float(((y.double() - ref.double()).abs() / beta).max())
        assert ratio <= 1.0, ratio
    # the bound is not vacuous: a small fraction of the value at the typical element
    assert float((beta / ref.double().abs().clamp_min(1e-3)).median()) < 1e-2


# ---------------------------------------------------------------------------------------------------- mistakes
def _trunc(t):
    """bf16 by truncation"""
    return (t.float().view(torch.int32) & ~0xFFFF).view(torch.float32)


def _round_to(t, bits):
    """round fp32 values to ``bits`` significant bits (nearest even)"""
    m, e = np.frexp(t.double().numpy())
    return torch.from_numpy(np.ldexp(np.round(np.ldexp(m, bits)), e - bits)).float()


SPLITS = {
    "split by truncation": lambda t: (_trunc(t), _trunc(t.float() - _trunc(t))),
    "lo from the unrounded hi": lambda t: (E.split(t)[0], E.split(t.float() - _trunc(t))[0]),
}


def _acc(a, w, kw, split=E.split, drop=None, accumulate=None):
    """the one-hot accumulator with a mistake: another split, a dropped term ("lo_hi": a_lo w_hi, "hi_lo": a_hi w_lo),
    or the sum of the terms rounded to ``accumulate`` bits (bf16: 8, TF32: 11)"""
    ah, al = (t.double() for t in split(a))
    wh, wl = (t.double() for t in split(w))
    terms = {"hi_hi": F.conv1d(ah, wh, **kw), "lo_hi": F.conv1d(al, wh, **kw), "hi_lo": F.conv1d(ah, wl, **kw)}
    out = terms["hi_hi"]
    for k in ("lo_hi", "hi_lo"):
        if k != drop:
            out = out + terms[k]
            if accumulate:
                out = _round_to(out, accumulate).double()
    return out


def _epi_mistake(acc, b, post, slope, res, scale, prev, mistake):
    v = acc.float().numpy() + b.numpy().reshape(1, -1, 1)
    act = (lambda t: np.where(t > 0, t, t * f32(slope))) if post == "lrelu" else (lambda t: t)
    if mistake == "bias after the activation":
        v = act(acc.float().numpy()) + b.numpy().reshape(1, -1, 1)
    else:
        v = act(v)
    s = f32(scale)
    r = res.numpy() if res is not None else f32(0)
    p = prev.numpy() if prev is not None else f32(0)
    if mistake == "out_scale before the residual":
        v = v * s + r
    else:
        v = v + r
        if mistake == "prev before out_scale":
            v = (v + p) * s
        elif mistake == "contracted scale and accumulate":
            v = (v.astype(np.float64) * float(s) + p.astype(np.float64)).astype(f32)
        else:
            v = v * s + p
    return torch.from_numpy(np.asarray(v, dtype=f32))


def _row(name, probe):
    d, kw, ref, _ = G.conv_case(name, probe)
    pl, pr = kw["padding"]
    a = E._pad(E.lrelu(d["x"], kw["pre_slope"]), pl, pr, kw["pad_mode"])
    ckw = dict(dilation=kw["dilation"], groups=kw["groups"])
    return d, kw, ref, a, ckw


def _differs(y, ref):
    ok = (y == ref) | (torch.isnan(y) & torch.isnan(ref))
    return int((~ok).sum())


# mistake: (row, probe) whose readback sees it
MISTAKES = {
    "split by truncation": ("tma_staged", "act"),
    "lo from the unrounded hi": ("tma_staged", "act"),
    "weight split by truncation": ("tma_staged", "w"),
    "a_lo w_hi dropped": ("register", "act"),
    "a_hi w_lo dropped": ("register", "w"),
    "bias after the activation": ("tma_staged", "act"),
    "out_scale before the residual": ("cpasync", "act"),
    "prev before out_scale": ("chunks", "act"),
    "contracted scale and accumulate": ("cpasync", "act"),
    "pre-slope after the split": ("reflect", "act"),
    "accumulation in bf16": ("tma_staged", "act"),
    "accumulation in TF32": ("tma_staged", "act"),
}


@pytest.mark.parametrize("mistake", list(MISTAKES))
def test_each_mistake_fails_a_readback(mistake):
    name, probe = MISTAKES[mistake]
    d, kw, ref, a, ckw = _row(name, probe)
    w = d["w"]
    epi = (d["b"], kw["post_act"], kw["post_slope"], d["res"], kw["out_scale"], d["prev"])
    assert torch.equal(_acc(a, w, ckw).float(), E.conv1d_acc(d["x"], w, **{k: kw[k] for k in
                       ("padding", "dilation", "groups", "pad_mode", "pre_slope")})[0].float())
    if mistake in SPLITS:
        acc = _acc(a, w, ckw, split=SPLITS[mistake])
    elif mistake == "weight split by truncation":
        acc = _acc(a, w, ckw, split=lambda t: SPLITS["split by truncation"](t) if t.shape == w.shape else E.split(t))
    elif mistake.endswith("dropped"):
        acc = _acc(a, w, ckw, drop="lo_hi" if mistake.startswith("a_lo") else "hi_lo")
    elif mistake == "pre-slope after the split":
        xp = E._pad(d["x"], *kw["padding"], kw["pad_mode"])
        acc = _acc(xp, w, ckw, split=lambda t: tuple(E.lrelu(p, kw["pre_slope"]) for p in E.split(t)) if t.shape == xp.shape
                   else E.split(t))
    elif mistake.startswith("accumulation"):
        acc = _acc(a, w, ckw, accumulate=8 if "bf16" in mistake else 11)
    else:
        acc = _acc(a, w, ckw)
        y = _epi_mistake(acc, *epi, mistake)
        assert torch.equal(_epi_mistake(acc, *epi, None), ref), "the mistake-free form is the emulation"
        assert _differs(y, ref) > 0, f"{mistake}: the readback of {name}/{probe} does not see it"
        return
    y = E.epilogue_f32(acc, *epi)
    assert _differs(y, ref) > 0, f"{mistake}: the readback of {name}/{probe} does not see it"


def test_accumulation_mistakes_also_leave_the_bound():
    """bf16 accumulation is also outside the bound on random data at a model shape (TF32 is seen by the readbacks)"""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(1, 64, 400, generator=g)
    w = torch.randn(64, 64, 7, generator=g) / math.sqrt(64 * 7)
    acc, mag, _ = E.conv1d_acc(x, w, padding=(9, 9), dilation=3, pre_slope=0.1)
    ref, beta = E.epilogue_f32(acc, err=E.accumulation_bound(mag, 3 * 64 * 7, E.U_TC))
    a = F.pad(E.lrelu(x, 0.1), (9, 9))
    ah, al = E.split(a)
    wh, wl = E.split(w)
    out = torch.zeros_like(ref, dtype=torch.float64)
    for ci in range(64):  # channel by channel, every partial sum rounded to bf16
        for t in (F.conv1d(ah[:, ci:ci + 1].double(), wh[:, ci:ci + 1].double(), dilation=3),
                  F.conv1d(al[:, ci:ci + 1].double(), wh[:, ci:ci + 1].double(), dilation=3),
                  F.conv1d(ah[:, ci:ci + 1].double(), wl[:, ci:ci + 1].double(), dilation=3)):
            out = _round_to(out + t, 8).double()
    assert float(((out - ref.double()).abs() / beta).max()) > 1.0


def test_readback_comparison_is_bitwise():
    """the readbacks tell -0 from +0 and accept any NaN where a NaN is expected"""
    ref = torch.tensor([0.0, 1.0, float("nan")])
    G._same(torch.tensor([0.0, 1.0, -float("nan")]), ref, "same")
    with pytest.raises(AssertionError):
        G._same(torch.tensor([-0.0, 1.0, float("nan")]), ref, "signed zero")
    with pytest.raises(AssertionError):
        G._same(torch.tensor([0.0, 1.0, 1.0]), ref, "NaN lost")
