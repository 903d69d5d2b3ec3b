"""How the convolutions round arbitrary fp32 values: the bf16 hi / lo split, the epilogue's order at the models' own
slopes and scales, and the size of the error on unstructured data (oracle/bf16x3.py, "rounding on fp32").

Readbacks (bit for bit, the sign of zero included; NaN where the reference is NaN): one operand is one-hot, so every
output element receives one non-zero (activation, weight) pair and the accumulator is hi + lo of the other operand,
exact in fp32.  Where one launch cannot read every input channel, a probe runs at several channel offsets, and each
row asserts that its launches together read every input channel.  The activation
probe drives arbitrary values through the loaders (TMA, cp.async, reflect / replicate / asymmetric padding, storage
offsets), the weight probe through the weight packers, and both through the epilogue, bit for bit against
``epilogue_f32``.  Every row reads its plan back (ops.PROFILE, pwgb_debug_get(1 / 2 / 3), ops.resblock_pair_plan), and
asserts the one-hot argument (``pair_count``) before it runs the GPU.

Bounds: on random-normal data at the models' shapes, |y - y_hat| <= beta at every element, y_hat the exact bf16x3 (or
fp32) products summed in fp64 and passed through ``epilogue_f32``, beta = (n - 1) u sum|terms| plus the epilogue's own
roundings.  The worst error / bound per case is printed, with the error against the fp64 conv of the fp32 operands
(reported, not asserted).  tests/test_conv_rounding_cpu.py checks the oracle and that each plausible mistake fails."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bf16x3 as E

pytestmark = pytest.mark.gpu

PLAN1 = ("MT", "na", "nb", "ns", "staged", "tma_act", "win_mode", "nco")
PLAN2 = ("nc", "tg", "ntg", "nsplit")
PLAN3 = ("kernel", "RCO", "WARPS_CO", "RT", "CI_T", "CO")
THIRD = float(np.float32(1.0 / 3.0))  # the MRF mean over three ResBlocks
SQRT_HALF = E.SQRT_HALF
WORST = {}


def _seed(name):
    return zlib.crc32(name.encode())


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    yield torch.device("cuda:0")
    if WORST:
        print(f"\n[conv_rounding] on {torch.cuda.get_device_name(0)}, worst error / bound, and max |y - fp64 conv| / peak:")
        for k, (r, t) in sorted(WORST.items()):
            print(f"  {k:28s} {r:.3e}   {t:.3e}")


def _lib():
    from parallelwavegan_b200 import capi

    return capi.lib()


def _readout(key, names):
    v = (C.c_int * len(names))()
    assert _lib().pwgb_debug_get(key, C.cast(v, C.c_void_p), C.sizeof(v)) == 0
    return dict(zip(names, list(v)))


def _profiled(fn, variant=0, engine=None):
    from parallelwavegan_b200 import ops

    old = ops.ENGINE
    ops.PROFILE = []
    _lib().pwgb_debug_set(1, variant)
    try:
        if engine is not None:
            ops.ENGINE = engine
        with torch.no_grad():
            y = fn()
        torch.cuda.synchronize()
        return y, [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None
        ops.ENGINE = old
        _lib().pwgb_debug_set(1, 0)


def _same(y, ref, what):
    """bit for bit (so -0 and +0 differ) wherever ref is a number, NaN (any payload) wherever ref is NaN"""
    y = y.detach().cpu()
    assert y.shape == ref.shape, (what, tuple(y.shape), tuple(ref.shape))
    ok = torch.where(torch.isnan(ref), torch.isnan(y), y.view(torch.int32) == ref.view(torch.int32))
    if bool(ok.all()):
        return
    bad = (~ok).nonzero()
    i = tuple(bad[0].tolist())
    raise AssertionError(f"{what}: {bad.shape[0]} of {ref.numel()} elements differ, first at {list(i)}: got "
                         f"{float(y[i])!r} ({y[i].view(torch.int32).item() & 0xFFFFFFFF:#010x}), expected {float(ref[i])!r} "
                         f"({ref[i].view(torch.int32).item() & 0xFFFFFFFF:#010x})")


def _d(t, dev):
    return None if t is None else t.to(dev)


def _at_offset(t, dev, off):
    buf = torch.empty(t.numel() + off, device=dev)
    v = buf[off:].view(t.shape)
    v.copy_(t)
    return v


def _exact(count, what):
    assert count <= 1.0, f"{what}: {count:.0f} non-zero pairs reach one output element, the probe is not one-hot"


def _channels(t):
    """the channels (dim 1) of t with a non-zero element"""
    return set((t != 0).transpose(0, 1).reshape(t.shape[1], -1).any(1).nonzero().reshape(-1).tolist())


def _weight_channels(w, groups):
    """the input channels a conv weight (cout, cin_g, K) reads through a non-zero element"""
    cout, cin_g = w.shape[0], w.shape[1]
    co, ci = (w != 0).any(2).nonzero(as_tuple=True)
    return set((co // (cout // groups) * cin_g + ci).tolist())


def _all_read(reads, n, what):
    assert reads == set(range(n)), f"{what}: the probe reads {len(reads)} of {n} input channels"


# ---------------------------------------------------------------------------------------------------- conv1d_tc readbacks
# name: (B, cin, cout, k, d, T, (pad_left, pad_right) or None for "same", pad_mode, groups, epilogue, options, plan)
#   epilogue: "plain" | "res" | "acc" | "both"; options: variant (2 = cp.async activations, 4 = register epilogue),
#   pre / post (lrelu slope 0.2) / scale, off (x storage offset), special (huge, inf and NaN inputs too)
CONV = {
    "tma_staged": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "both", dict(post=0.2), dict(MT=2, staged=1, tma_act=1)),
    "register": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "both", dict(post=0.2, variant=4), dict(MT=2, staged=0)),
    "cpasync": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "both", dict(variant=2, scale=SQRT_HALF),
                dict(MT=2, staged=1, tma_act=0)),
    "reflect": (2, 64, 32, 7, 3, 2052, None, "reflect", 1, "res", dict(pre=0.2), dict(MT=2, staged=1, tma_act=0)),
    "replicate": (2, 32, 64, 7, 1, 2052, (5, 1), "replicate", 1, "plain", dict(post=0.2), dict(MT=2, staged=0, tma_act=0)),
    "asymmetric": (2, 32, 32, 5, 2, 2052, (8, 0), "zero", 1, "both", {}, dict(MT=2, staged=1, tma_act=1)),
    "x_offset": (2, 32, 32, 3, 1, 2052, None, "zero", 1, "both", dict(off=1), dict(MT=2, staged=1, tma_act=0)),
    "chunks": (2, 64, 256, 3, 1, 1028, None, "zero", 1, "acc", dict(scale=SQRT_HALF), dict(MT=1, staged=1, nco=2)),
    "chunks_register": (1, 64, 256, 3, 1, 1028, None, "zero", 1, "both", dict(variant=4), dict(MT=1, staged=0, nco=2)),
    "groups16": (1, 512, 256, 41, 1, 1024, None, "zero", 16, "acc", dict(post=0.2), dict(MT=2, staged=1, nco=16)),
    "special": (2, 64, 96, 3, 1, 132, None, "zero", 1, "both", dict(special=True), dict(MT=1, staged=1)),
    "special_register": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "both", dict(special=True, variant=4), dict(MT=2, staged=0)),
}
PROBES = ("act", "w")


def _pads(k, d, pad):
    return pad or ((k - 1) // 2 * d, (k - 1) // 2 * d)


def _conv_w_probe(T, k, d, pl, pr):
    """(spacing, margin) of the weight probe's one-hot input"""
    return (k - 1) * d + 1, max(pl, pr) + 1


def conv_offsets(name, probe):
    """the channel offsets of the launches that together read every input channel of row ``name``"""
    B, cin, cout, k, d, T, pad, mode, groups, *_ = CONV[name]
    if probe == "act":
        return E.probe_offsets(cout // groups, cin // groups)
    return E.probe_offsets(len(E.onehot_positions(T, *_conv_w_probe(T, k, d, *_pads(k, d, pad)))), cin // groups)


def conv_case(name, probe, offset=0):
    """the inputs of row ``name`` under ``probe`` ("act": arbitrary x, one-hot weights; "w": one-hot x, arbitrary
    weights) at channel ``offset``, its keyword arguments, the expected output and the input channels it reads;
    asserts the one-hot argument"""
    B, cin, cout, k, d, T, pad, mode, groups, epi, opt, _ = CONV[name]
    pl, pr = _pads(k, d, pad)
    t_out = T + pl + pr - (k - 1) * d
    s = _seed(name + probe) + offset
    if probe == "act":
        x = E.fp32_values((B, cin, T), s, special=opt.get("special", False))
        w = E.onehot_weight(cout, cin // groups, k, offset)
        reads = _weight_channels(w, groups)
    else:
        x = E.onehot_input(B, cin, T, *_conv_w_probe(T, k, d, pl, pr), groups, offset)
        w = E.fp32_values((cout, cin // groups, k), s)
        reads = _channels(x)
    bias = E.fp32_values((cout,), s + 1)
    res = E.fp32_values((B, cout, t_out), s + 2) if epi in ("res", "both") else None
    prev = E.fp32_values((B, cout, t_out), s + 3) if epi in ("acc", "both") else None
    pre = opt.get("pre", 0.1)
    kw = dict(padding=(pl, pr), dilation=d, groups=groups, pad_mode=mode, pre_slope=pre,
              post_act="lrelu" if "post" in opt else None, post_slope=opt.get("post", 0.0), out_scale=opt.get("scale", THIRD))
    _exact(E.pair_count(lambda a, b: F.conv1d(E._pad(a, pl, pr, mode), b, dilation=d, groups=groups), x, w), name)
    if opt.get("special"):
        acc = E.conv1d_acc_ieee(x, w, padding=(pl, pr), dilation=d, groups=groups, pad_mode=mode, pre_slope=pre)
    else:
        acc = E.conv1d_acc(x, w, padding=(pl, pr), dilation=d, groups=groups, pad_mode=mode, pre_slope=pre)[0]
    ref = E.epilogue_f32(acc, bias, kw["post_act"], kw["post_slope"], res, kw["out_scale"], prev)
    return dict(x=x, w=w, b=bias, res=res, prev=prev), kw, ref, reads


@pytest.mark.parametrize("probe", PROBES)
@pytest.mark.parametrize("name", list(CONV))
def test_conv1d_tc_readback(dev, name, probe):
    from parallelwavegan_b200 import ops

    cin, opt, plan = CONV[name][1], CONV[name][10], CONV[name][11]
    reads = set()
    for offset in conv_offsets(name, probe):
        d, kw, ref, r = conv_case(name, probe, offset)
        reads |= r
        xd = _at_offset(d["x"], dev, opt["off"]) if opt.get("off") else d["x"].to(dev)
        out = _d(d["prev"], dev)
        y, names = _profiled(lambda: ops.conv1d(xd, d["w"].to(dev), d["b"].to(dev), residual=_d(d["res"], dev), out=out,
                                                accumulate=out is not None, **kw), opt.get("variant", 0))
        got = _readout(1, PLAN1)
        assert names == ["conv1d_tc"], names
        assert {k: got[k] for k in plan} == plan, got
        _same(y, ref, f"{name}/{probe} offset {offset}")
    _all_read(reads, cin, f"{name}/{probe}")


# tanh is not correctly rounded: its value is checked within libdevice's 2 ulp of tanh, and the steps around it exactly
TANH = {"tanh_staged": ("tma_staged", dict(MT=2, staged=1)), "tanh_register": ("register", dict(MT=2, staged=0))}


@pytest.mark.parametrize("name", list(TANH))
def test_conv1d_tc_tanh(dev, name):
    from parallelwavegan_b200 import ops

    row, plan = TANH[name]
    opt = CONV[row][10]
    d, kw, _, _ = conv_case(row, "act")
    kw = dict(kw, post_act="tanh")
    acc = E.conv1d_acc(d["x"], d["w"], **{k: kw[k] for k in ("padding", "dilation", "groups", "pad_mode", "pre_slope")})[0]
    x, w, b = d["x"].to(dev), d["w"].to(dev), d["b"].to(dev)
    t, names = _profiled(lambda: ops.conv1d(x, w, b, **dict(kw, out_scale=1.0)), opt.get("variant", 0))
    assert names == ["conv1d_tc"], names
    t = t.cpu()
    v = E.epilogue_f32(acc, d["b"]).double()  # tanh's argument, exact
    ulp = torch.from_numpy(np.spacing(np.abs(np.tanh(v.numpy())).astype(np.float32))).double()
    err = (t.double() - torch.tanh(v)).abs()
    assert bool((err <= 2 * ulp).all()), f"{name}: tanh {float((err / ulp).max()):.2f} ulp from tanh"
    out = d["prev"].to(dev)
    y, names = _profiled(lambda: ops.conv1d(x, w, b, residual=d["res"].to(dev), out=out, accumulate=True, **kw),
                         opt.get("variant", 0))
    got = _readout(1, PLAN1)
    assert {k: got[k] for k in plan} == plan, got
    _same(y, E.epilogue_f32(acc, d["b"], "tanh", 0.0, d["res"], kw["out_scale"], d["prev"], tanh=t.numpy()), name)


# ---------------------------------------------------------------------------------------------------- fused ResBlock pair
# name: (C, k, d, mode) at B = 1, T = 1028, slope 0.1; "acc" accumulates with out_scale 1/3 (the MRF mean)
PAIR = {"c32_k3_d1": (32, 3, 1, "acc"), "c32_k11_d5": (32, 11, 5, "plain"), "c64_k7_d3": (64, 7, 3, "acc"),
        "c64_k11_d5": (64, 11, 5, "plain")}
PAIR_PROBES = ("act", "w1", "w2")


def _pair_w_probe(k, d):
    """(spacing, margin) of the pair's one-hot input: beyond both convs' receptive fields"""
    return 2 * ((k - 1) * d + k), (k - 1) // 2 * (d + 1) + 1


def pair_offsets(name, probe, T=1028):
    Cc, k, d, _ = PAIR[name]
    return [0] if probe == "act" else E.probe_offsets(len(E.onehot_positions(T, *_pair_w_probe(k, d))), Cc)


def pair_case(name, probe, offset=0, T=1028, B=1):
    """act: arbitrary x, both convs one-hot; w1: one-hot x, arbitrary conv1; w2: one-hot x and conv1 with b1 = 0 (so
    h is one-hot), arbitrary conv2.  Returns the inputs, the expected output and the input channels read."""
    Cc, k, d, mode = PAIR[name]
    s = _seed(name + probe) + offset
    p1, p2 = (k - 1) // 2 * d, (k - 1) // 2
    if probe == "act":
        x = E.fp32_values((B, Cc, T), s)
    else:
        x = E.onehot_input(B, Cc, T, *_pair_w_probe(k, d), offset=offset)
    w1 = E.fp32_values((Cc, Cc, k), s + 1) if probe == "w1" else E.onehot_weight(Cc, Cc, k)
    w2 = E.fp32_values((Cc, Cc, k), s + 2) if probe == "w2" else E.onehot_weight(Cc, Cc, k)
    b1 = torch.zeros(Cc) if probe == "w2" else E.fp32_values((Cc,), s + 3)
    b2 = E.fp32_values((Cc,), s + 4)
    prev = E.fp32_values((B, Cc, T), s + 5) if mode == "acc" else None
    scale = THIRD if mode == "acc" else 1.0
    _exact(E.pair_count(lambda a, b: F.conv1d(a, b, padding=p1, dilation=d), x, w1), name + " conv1")
    acc1 = E.conv1d_acc(x, w1, padding=(p1, p1), dilation=d, pre_slope=0.1)[0]
    h = E.epilogue_f32(acc1, b1)
    _exact(E.pair_count(lambda a, b: F.conv1d(a, b, padding=p2), h, w2), name + " conv2")
    acc2 = E.conv1d_acc(h, w2, padding=(p2, p2), pre_slope=0.1)[0]
    ref = E.epilogue_f32(acc2, b2, residual=x, out_scale=scale, prev=prev)
    reads = _weight_channels(w1, 1) if probe == "act" else _channels(x)
    return dict(x=x, w1=w1, b1=b1, w2=w2, b2=b2, prev=prev, scale=scale), ref, reads


def _run_pair(dev, name, d):
    from parallelwavegan_b200 import ops

    Cc, k, dil, mode = PAIR[name]
    B, _, T = d["x"].shape
    plan = ops.resblock_pair_plan(Cc, T, k, dil, batch=B)
    assert plan is not None and plan["TT"] == (256 if Cc == 32 else 128), plan
    out = _d(d["prev"], dev)
    y, names = _profiled(lambda: ops.resblock_pair(*(d[n].to(dev) for n in ("x", "w1", "b1", "w2", "b2")), kernel_size=k,
                                                   dilation=dil, slope=0.1, out=out, accumulate=out is not None,
                                                   out_scale=d["scale"]))
    assert names == ["resblock_pair_tc"], names
    return y


@pytest.mark.parametrize("probe", PAIR_PROBES)
@pytest.mark.parametrize("name", list(PAIR))
def test_resblock_pair_readback(dev, name, probe):
    reads = set()
    for offset in pair_offsets(name, probe):
        d, ref, r = pair_case(name, probe, offset)
        reads |= r
        _same(_run_pair(dev, name, d), ref, f"pair {name}/{probe} offset {offset}")
    _all_read(reads, PAIR[name][0], f"pair {name}/{probe}")


# ---------------------------------------------------------------------------------------------------- conv-transpose
# name: (B, cin1, cin2, cout, K, stride, padding, output_padding, t_in, plan or None); cin2 > 0: the two-source entry
CONVTR = {
    "up0_512_256_k16s8": (1, 512, 0, 256, 16, 8, 4, 0, 32, dict(MT=1, nco=16)),
    "up3_64_32_k4s2": (2, 64, 0, 32, 4, 2, 1, 0, 1024, dict(MT=2, nco=1)),
    "cat_128_128_64_k10s5": (2, 128, 128, 64, 10, 5, 3, 1, 480, dict(MT=1, staged=0, tma_act=1, nco=4)),
}


def convtr_offsets(row, probe):
    B, cin1, cin2, cout, K, s, p, op, t_in, _ = row
    return [0] if probe == "act" else E.probe_offsets(len(E.onehot_positions(t_in, -(-K // s) + 1, 0)), cin1 + cin2)


def convtr_case(name, probe, offset=0, bf16x3=True, row=None):
    """act: arbitrary x, every input channel (of both sources) read through one tap per phase; w: one-hot x, arbitrary
    w.  Returns x, w, b, the keyword arguments, the expected output and the input channels read."""
    B, cin1, cin2, cout, K, s, p, op, t_in, _ = row or CONVTR[name]
    cin = cin1 + cin2
    sd = _seed(name + probe) + offset
    if probe == "act":
        x = E.fp32_values((B, cin, t_in), sd)
        w = E.onehot_weight_transposed(cin, cout, K, s)
        reads = set((w != 0).any(2).any(1).nonzero().reshape(-1).tolist())
    else:
        x = E.onehot_input(B, cin, t_in, -(-K // s) + 1, 0, offset=offset)
        w = E.fp32_values((cin, cout, K), sd)
        reads = _channels(x)
    b = E.fp32_values((cout,), sd + 1)
    kw = dict(stride=s, padding=p, output_padding=op)
    _exact(E.pair_count(lambda a, c: F.conv_transpose1d(a, c, **kw), x, w), name)
    acc = E.conv_transpose1d_acc(x, w, pre_slope=0.1, bf16x3=bf16x3, **kw)[0]
    return x, w, b, kw, E.epilogue_f32(acc, b), reads


@pytest.mark.parametrize("probe", PROBES)
@pytest.mark.parametrize("name", list(CONVTR))
def test_conv_transpose1d_tc_readback(dev, name, probe):
    from parallelwavegan_b200 import ops

    cin1, cin2 = CONVTR[name][1], CONVTR[name][2]
    plan = CONVTR[name][-1]
    reads = set()
    for offset in convtr_offsets(CONVTR[name], probe):
        x, w, b, kw, ref, r = convtr_case(name, probe, offset)
        reads |= r
        xd, wd, bd = x.to(dev), w.to(dev), b.to(dev)
        if cin2:
            y, names = _profiled(lambda: ops.conv_transpose1d_cat(xd[:, :cin1].contiguous(), xd[:, cin1:].contiguous(), wd, bd,
                                                                  pre_slope=0.1, **kw))
            assert names == ["conv_transpose1d_cat"], names
        else:
            y, names = _profiled(lambda: ops.conv_transpose1d(xd, wd, bd, pre_slope=0.1, **kw))
            assert names == ["conv_transpose1d"], names
        got = _readout(1, PLAN1)
        assert {k: got[k] for k in plan} == plan, got
        _same(y, ref, f"{name}/{probe} offset {offset}")
    _all_read(reads, cin1 + cin2, f"{name}/{probe}")


# ---------------------------------------------------------------------------------------------------- strided (s2d)
# name: (cin, cout, K, stride, groups, pad, rows, period, B, plan) with post lrelu 0.1, the discriminators' slope
STRIDED = {"msd_k41_s4_g16": (256, 512, 41, 4, 16, 20, 1024, 1, 2, dict(MT=2, staged=0, tma_act=0, nco=16)),
           "mpd_p5_l2": (32, 128, 5, 3, 1, 2, 273, 5, 2, dict(MT=1, staged=0, tma_act=1, nco=1))}


def strided_offsets(name, probe):
    cin, cout, K, s, G, pad, rows, P, B = STRIDED[name][:9]
    if probe == "act":
        return E.probe_offsets(cout // G, cin // G)
    return E.probe_offsets(len(E.onehot_positions(rows, K, pad + 1)), cin // G)


def strided_case(name, probe, offset=0):
    """x, w, b, the expected output and the input channels read"""
    cin, cout, K, s, G, pad, rows, P, B = STRIDED[name][:9]
    sd = _seed(name + probe) + offset
    if probe == "act":
        x, w = E.fp32_values((B, cin, rows * P), sd), E.onehot_weight(cout, cin // G, K, offset)
        reads = _weight_channels(w, G)
    else:
        x = E.onehot_input(B * P, cin, rows, K, pad + 1, G, offset).view(B, P, cin, rows).permute(0, 2, 3, 1)
        x = x.reshape(B, cin, rows * P)
        w = E.fp32_values((cout, cin // G, K), sd)
        reads = _channels(x)
    b = E.fp32_values((cout,), sd + 1)
    xc = x.view(B, cin, rows, P).permute(0, 3, 1, 2).reshape(B * P, cin, rows)
    _exact(E.pair_count(lambda a, c: F.conv1d(a, c, stride=s, padding=pad, groups=G), xc, w), name)
    acc = E.conv1d_acc(xc, w, stride=s, padding=(pad, pad), groups=G)[0]
    ref = E.epilogue_f32(acc, b, "lrelu", 0.1).view(B, P, cout, -1).permute(0, 2, 3, 1)
    return x, w, b, (ref if P > 1 else ref[..., 0]).contiguous(), reads


@pytest.mark.parametrize("probe", PROBES)
@pytest.mark.parametrize("name", list(STRIDED))
def test_strided_conv_tc_readback(dev, name, probe):
    from parallelwavegan_b200 import ops

    cin, cout, K, s, G, pad, rows, P, B, plan = STRIDED[name]
    reads = set()
    for offset in strided_offsets(name, probe):
        x, w, b, ref, r = strided_case(name, probe, offset)
        reads |= r
        xd = x.to(dev) if P == 1 else x.to(dev).view(B, cin, rows, P)
        wd = w.to(dev) if P == 1 else w.to(dev).unsqueeze(-1)
        y, names = _profiled(lambda: ops.conv1d(xd, wd, b.to(dev), stride=s, padding=pad, groups=G, period=P, post_act="lrelu",
                                                post_slope=0.1))
        assert names == ["s2d", "conv1d_tc"], names
        got = _readout(1, PLAN1)
        assert {k: got[k] for k in plan} == plan, got
        _same(y, ref, f"{name}/{probe} offset {offset}")
    _all_read(reads, cin, f"{name}/{probe}")


# ---------------------------------------------------------------------------------------------------- weight gradient
# name: (B, cin, cout, k, d, pad, T, groups, x_slope, g_slope, plan)
WGRAD = {
    "ntg3_k11": (2, 32, 64, 11, 1, 5, 1024, 1, 0.1, 0.2, dict(nc=32, tg=4, ntg=3, nsplit=2)),
    "groups4": (2, 128, 128, 5, 1, 2, 1024, 4, 0.2, 0.1, dict(nc=32, tg=4, ntg=2, nsplit=2)),
    "nc64_k1": (2, 64, 64, 1, 1, 0, 1024, 1, 0.1, 0.1, dict(nc=64, tg=1, ntg=1, nsplit=2)),
}
WGRAD_PROBES = ("x", "gy")


def wgrad_case(name, probe):
    """x: gy one-hot (one time step per output channel, in batch 0), arbitrary x; gy: x one-hot (one time step per
    input channel), arbitrary gy"""
    B, cin, cout, k, d, pad, T, G, xs, gs, _ = WGRAD[name]
    t_out = T + 2 * pad - (k - 1) * d
    sd = _seed(name + probe)
    if probe == "x":
        x = E.fp32_values((B, cin, T), sd)
        gy = torch.zeros(B, cout, t_out)
        co = torch.arange(cout)
        gy[0, co, (co * 37) % t_out] = 1.0
    else:
        gy = E.fp32_values((B, cout, t_out), sd)
        x = torch.zeros(B, cin, T)
        ci = torch.arange(cin)
        x[0, ci, (ci * 29) % T] = 1.0

    def wg(a, g):
        ap = F.pad(a, (pad, pad))
        return torch.nn.grad.conv1d_weight(ap, (cout, cin // G, k), g, dilation=d, groups=G)

    _exact(E.pair_count(lambda a, g: wg(a, g), x, gy), name)
    acc = E.conv1d_wgrad_acc(x, gy, k, pad_left=pad, dilation=d, groups=G, x_slope=xs, g_slope=gs)[0]
    return x, gy, E.epilogue_f32(acc)


@pytest.mark.parametrize("probe", WGRAD_PROBES)
@pytest.mark.parametrize("name", list(WGRAD))
def test_conv1d_wgrad_tc_readback(dev, name, probe):
    from parallelwavegan_b200 import ops

    B, cin, cout, k, d, pad, T, G, xs, gs, plan = WGRAD[name]
    x, gy, ref = wgrad_case(name, probe)
    dw, names = _profiled(lambda: ops.conv1d_wgrad(x.to(dev), gy.to(dev), (cout, cin // G, k), padding=pad, dilation=d,
                                                   groups=G, x_slope=xs, g_slope=gs))
    assert names == ["conv1d_wgrad_tc"], names
    assert _readout(2, PLAN2) == plan
    _same(dw, ref, f"{name}/{probe}")


# ---------------------------------------------------------------------------------------------------- FFMA engine
# no split: the accumulator is the activated input itself, so these check the FFMA epilogue's order and pre-activation.
# name: (B, cin, cout, K, T, pad, mode, epilogue, options, plan)
FFMA = {
    "g88_rt4": (2, 16, 64, 3, 700, (1, 1), "zero", "both", dict(post=0.2), dict(kernel=0, RCO=8, WARPS_CO=8, RT=4, CI_T=16)),
    "g84_rt4_special": (2, 24, 40, 5, 1025, (2, 2), "zero", "both", dict(special=True, scale=SQRT_HALF),
                        dict(kernel=0, RCO=8, WARPS_CO=4, RT=4, CI_T=16)),
    "g41_rt1_replicate": (2, 8, 4, 3, 300, (2, 1), "replicate", "res", {}, dict(kernel=0, RCO=4, WARPS_CO=1, RT=1)),
    "fc2_reflect": (2, 16, 2, 5, 4096, (2, 2), "reflect", "plain", dict(post=0.2), dict(kernel=2, CO=2)),
}


@pytest.mark.parametrize("name", list(FFMA))
def test_conv1d_ffma_readback(dev, name):
    from parallelwavegan_b200 import ops

    B, cin, cout, K, T, (pl, pr), mode, epi, opt, plan = FFMA[name]
    t_out = T + pl + pr - (K - 1)
    reads = set()
    for offset in E.probe_offsets(cout, cin):
        s = _seed(name) + offset
        x, w = E.fp32_values((B, cin, T), s, special=opt.get("special", False)), E.onehot_weight(cout, cin, K, offset)
        reads |= _weight_channels(w, 1)
        b = E.fp32_values((cout,), s + 1)
        res = E.fp32_values((B, cout, t_out), s + 2) if epi in ("res", "both") else None
        prev = E.fp32_values((B, cout, t_out), s + 3) if epi in ("acc", "both") else None
        kw = dict(padding=(pl, pr), pad_mode=mode, pre_slope=0.2, post_act="lrelu" if "post" in opt else None,
                  post_slope=opt.get("post", 0.0), out_scale=opt.get("scale", THIRD))
        _exact(E.pair_count(lambda a, c: F.conv1d(E._pad(a, pl, pr, mode), c), x, w), name)
        acc = E.conv1d_acc_ieee(x, w, padding=(pl, pr), pad_mode=mode, pre_slope=0.2, bf16x3=False)
        ref = E.epilogue_f32(acc, b, kw["post_act"], kw["post_slope"], res, kw["out_scale"], prev)
        out = _d(prev, dev)
        y, names = _profiled(lambda: ops.conv1d_raw(x.to(dev), w.to(dev), b.to(dev), residual=_d(res, dev), out=out,
                                                    accumulate=out is not None, **kw), engine="simt")
        assert names == ["conv1d"], names
        got = _readout(3, PLAN3)
        assert {k: got[k] for k in plan} == plan, got
        _same(y, ref, f"{name} offset {offset}")
    _all_read(reads, cin, name)


FFMA_CONVTR = {"ct_cin20": ((2, 20, 0, 16, 4, 2, 1, 1, 200, None), dict(kernel=0, RCO=8, WARPS_CO=4, RT=4))}


@pytest.mark.parametrize("probe", PROBES)
@pytest.mark.parametrize("name", list(FFMA_CONVTR))
def test_conv_transpose1d_ffma_readback(dev, name, probe):
    from parallelwavegan_b200 import ops

    row, plan = FFMA_CONVTR[name]
    reads = set()
    for offset in convtr_offsets(row, probe):
        x, w, b, kw, ref, r = convtr_case(name, probe, offset, bf16x3=False, row=row)
        reads |= r
        y, names = _profiled(lambda: ops.conv_transpose1d_raw(x.to(dev), w.to(dev), b.to(dev), pre_slope=0.1, **kw),
                             engine="simt")
        assert names == ["conv_transpose1d"], names
        got = _readout(3, PLAN3)
        assert {k: got[k] for k in plan} == plan, got
        _same(y, ref, f"{name}/{probe} offset {offset}")
    _all_read(reads, row[1] + row[2], f"{name}/{probe}")


# ---------------------------------------------------------------------------------------------------- bounds
def _randn(shape, seed, scale=1.0):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * scale


def _record(name, y, ref, beta, true):
    y = y.detach().cpu().double()
    assert y.shape == ref.shape, (name, tuple(y.shape), tuple(ref.shape))
    assert bool(torch.isfinite(y).all()), name
    err = (y - ref.double()).abs()
    r = float((err / beta).max())
    t = float((y - true).abs().max() / true.abs().max())
    WORST[name] = (r, t)
    assert r <= 1.0, f"{name}: error {r:.3f} x the bound"


def _epi64(acc, bias=None, post=None, slope=0.0, res=None, scale=1.0, prev=None):
    """the epilogue in fp64 (the value a user means by the conv)"""
    v = acc + (0 if bias is None else bias.double().reshape(1, -1, *([1] * (acc.dim() - 2))))
    if post == "lrelu":
        v = torch.where(v > 0, v, v * slope)
    elif post == "tanh":
        v = torch.tanh(v)
    if res is not None:
        v = v + res.double()
    v = v * scale
    return v if prev is None else v + prev.double()


# name: (B, cin, cout, K, d, T, pad_mode, pre, post, epilogue, scale)
BOUND_CONV = {
    "hifigan_in_80_512_k7": (2, 80, 512, 7, 1, 256, "zero", 1.0, None, "plain", 1.0),
    "resblock_256_k3_d1": (2, 256, 256, 3, 1, 2048, "zero", 0.1, None, "res", 1.0),
    "resblock_128_k7_d3": (2, 128, 128, 7, 3, 4096, "zero", 0.1, None, "plain", 1.0),
    "resblock_64_k11_d5": (1, 64, 64, 11, 5, 8192, "zero", 0.1, None, "both", THIRD),
    "hifigan_out_32_1_k7": (1, 32, 1, 7, 1, 16384, "zero", 0.1, "tanh", "plain", 1.0),
    "melgan_256_k3_d9_reflect": (2, 256, 256, 3, 9, 2048, "reflect", 0.2, None, "res", 1.0),
    "melgan_in_80_512_k7_reflect": (2, 80, 512, 7, 1, 256, "reflect", 1.0, None, "plain", 1.0),
}


@pytest.mark.parametrize("name", list(BOUND_CONV))
def test_conv1d_bound(dev, name):
    from parallelwavegan_b200 import ops

    B, cin, cout, K, d, T, mode, pre, post, epi, scale = BOUND_CONV[name]
    s = _seed(name)
    x, w, b = _randn((B, cin, T), s), _randn((cout, cin, K), s + 1, 1 / math.sqrt(cin * K)), _randn((cout,), s + 2, 0.1)
    res = _randn((B, cout, T), s + 3) if epi in ("res", "both") else None
    prev = _randn((B, cout, T), s + 4) if epi in ("acc", "both") else None
    p = (K - 1) // 2 * d
    out = _d(prev, dev)
    y, names = _profiled(lambda: ops.conv1d(x.to(dev), w.to(dev), b.to(dev), padding=p, dilation=d, pad_mode=mode, pre_slope=pre,
                                            post_act=post, post_slope=0.0, residual=_d(res, dev), out_scale=scale, out=out,
                                            accumulate=out is not None))
    tc = names == ["conv1d_tc"]
    assert names in (["conv1d_tc"], ["conv1d"]), names
    acc, mag, _ = E.conv1d_acc(x, w, padding=(p, p), dilation=d, pad_mode=mode, pre_slope=pre, bf16x3=tc)
    # FFMA: n fmas, each rounding once (the first one rounds the product); tensor cores: exact products, n - 1 additions
    n = 3 * cin * K if tc else cin * K + 1
    ref, beta = E.epilogue_f32(acc, b, post, 0.0, res, scale, prev, err=E.accumulation_bound(mag, n, E.U_TC if tc else E.U_FFMA))
    a = E._pad(E.lrelu(x, pre).double(), p, p, mode)
    true = _epi64(F.conv1d(a, w.double(), dilation=d), b, post, 0.0, res, scale, prev)
    _record(name + ("" if tc else " (ffma)"), y, ref, beta, true)


# name: (C, k, d, T, mode)
BOUND_PAIR = {"pair_64_k3_d1": (64, 3, 1, 8192, "acc"), "pair_64_k11_d5": (64, 11, 5, 8192, "plain"),
              "pair_32_k7_d3": (32, 7, 3, 16384, "acc")}


@pytest.mark.parametrize("name", list(BOUND_PAIR))
def test_resblock_pair_bound(dev, name):
    from parallelwavegan_b200 import ops

    Cc, k, d, T, mode = BOUND_PAIR[name]
    s = _seed(name)
    x = _randn((1, Cc, T), s)
    w1, w2 = _randn((Cc, Cc, k), s + 1, 1 / math.sqrt(Cc * k)), _randn((Cc, Cc, k), s + 2, 1 / math.sqrt(Cc * k))
    b1, b2 = _randn((Cc,), s + 3, 0.1), _randn((Cc,), s + 4, 0.1)
    prev = _randn((1, Cc, T), s + 5) if mode == "acc" else None
    scale = THIRD if mode == "acc" else 1.0
    out = _d(prev, dev)
    y, names = _profiled(lambda: ops.resblock_pair(x.to(dev), w1.to(dev), b1.to(dev), w2.to(dev), b2.to(dev), kernel_size=k,
                                                   dilation=d, slope=0.1, out=out, accumulate=out is not None, out_scale=scale))
    assert names == ["resblock_pair_tc"], names
    n = 3 * Cc * k
    p1, p2 = (k - 1) // 2 * d, (k - 1) // 2
    acc1, mag1, _ = E.conv1d_acc(x, w1, padding=(p1, p1), dilation=d, pre_slope=0.1)
    h, e_h = E.epilogue_f32(acc1, b1, err=E.accumulation_bound(mag1, n, E.U_TC))
    # conv2's operand: lrelu(h) (1-Lipschitz, one rounding), then the split of a value within e of lrelu(h)
    ha = E.lrelu(h, 0.1).double()
    e_a = e_h + E.U_FFMA * ha.abs() + E.SUBNORMAL
    e_op = E.split_bound(ha, e_a) + E.split_bound(ha, torch.zeros_like(ha))
    acc2, mag2, _ = E.conv1d_acc(h, w2, padding=(p2, p2), pre_slope=0.1)
    wabs = w2.double().abs() * (1 + 2.0 ** -8)
    e_acc2 = F.conv1d(e_op, wabs, padding=p2) + E.accumulation_bound(mag2 + F.conv1d(e_op, wabs, padding=p2), n, E.U_TC)
    ref, beta = E.epilogue_f32(acc2, b2, residual=x, out_scale=scale, prev=prev, err=e_acc2)
    h64 = _epi64(F.conv1d(E.lrelu(x, 0.1).double(), w1.double(), padding=p1, dilation=d), b1)
    true = _epi64(F.conv1d(torch.where(h64 > 0, h64, 0.1 * h64), w2.double(), padding=p2), b2, res=x, scale=scale, prev=prev)
    _record(name, y, ref, beta, true)


# name: (B, cin, cout, K, stride, padding, t_in)
BOUND_CONVTR = {"up_512_256_k16_s8": (1, 512, 256, 16, 8, 4, 256), "up_64_32_k4_s2": (2, 64, 32, 4, 2, 1, 8192)}


@pytest.mark.parametrize("name", list(BOUND_CONVTR))
def test_conv_transpose1d_bound(dev, name):
    from parallelwavegan_b200 import ops

    B, cin, cout, K, st, p, t_in = BOUND_CONVTR[name]
    s = _seed(name)
    x, w, b = _randn((B, cin, t_in), s), _randn((cin, cout, K), s + 1, 1 / math.sqrt(cin * K / st)), _randn((cout,), s + 2, 0.1)
    y, names = _profiled(lambda: ops.conv_transpose1d(x.to(dev), w.to(dev), b.to(dev), stride=st, padding=p, pre_slope=0.1))
    assert names == ["conv_transpose1d"], names
    acc, mag, _ = E.conv_transpose1d_acc(x, w, stride=st, padding=p, pre_slope=0.1)
    ref, beta = E.epilogue_f32(acc, b, err=E.accumulation_bound(mag, 3 * cin * -(-K // st), E.U_TC))
    true = _epi64(F.conv_transpose1d(E.lrelu(x, 0.1).double(), w.double(), stride=st, padding=p), b)
    _record(name, y, ref, beta, true)


# name: (cin, cout, K, stride, groups, pad, rows, period, B)
BOUND_STRIDED = {"msd_k41_s4_g16": (256, 512, 41, 4, 16, 20, 2048, 1, 2), "mpd_p3_l2": (32, 128, 5, 3, 1, 2, 2731, 3, 2)}


@pytest.mark.parametrize("name", list(BOUND_STRIDED))
def test_strided_conv_bound(dev, name):
    from parallelwavegan_b200 import ops

    cin, cout, K, st, G, pad, rows, P, B = BOUND_STRIDED[name]
    s = _seed(name)
    x, w, b = _randn((B, cin, rows * P), s), _randn((cout, cin // G, K), s + 1, 1 / math.sqrt(cin // G * K)), _randn((cout,), s + 2, 0.1)
    xd = x.to(dev) if P == 1 else x.to(dev).view(B, cin, rows, P)
    wd = w.to(dev) if P == 1 else w.to(dev).unsqueeze(-1)
    y, names = _profiled(lambda: ops.conv1d(xd, wd, b.to(dev), stride=st, padding=pad, groups=G, period=P, post_act="lrelu",
                                            post_slope=0.1))
    assert names == ["s2d", "conv1d_tc"], names
    xc = x.view(B, cin, rows, P).permute(0, 3, 1, 2).reshape(B * P, cin, rows)
    acc, mag, _ = E.conv1d_acc(xc, w, stride=st, padding=(pad, pad), groups=G)
    ref, beta = E.epilogue_f32(acc, b, "lrelu", 0.1, err=E.accumulation_bound(mag, 3 * cin // G * K, E.U_TC))
    true = _epi64(F.conv1d(xc.double(), w.double(), stride=st, padding=pad, groups=G), b, "lrelu", 0.1)

    def view(t):
        t = t.reshape(B, P, cout, -1).permute(0, 2, 3, 1)
        return (t if P > 1 else t[..., 0]).contiguous()

    _record(name, y, view(ref), view(beta), view(true))


# name: (B, cin, cout, k, d, pad, T, groups, x_slope, g_slope): the ResBlock convs' weight gradients of a training step
BOUND_WGRAD = {"wgrad_128_k7_d3": (4, 128, 128, 7, 3, 9, 8192, 1, 0.1, 1.0),
               "wgrad_256_k3_d1": (4, 256, 256, 3, 1, 1, 4096, 1, 0.1, 1.0),
               "wgrad_64_k11_d5": (4, 64, 64, 11, 5, 25, 16384, 1, 0.2, 0.2)}


@pytest.mark.parametrize("name", list(BOUND_WGRAD))
def test_conv1d_wgrad_bound(dev, name):
    from parallelwavegan_b200 import ops

    B, cin, cout, k, d, pad, T, G, xs, gs = BOUND_WGRAD[name]
    t_out = T + 2 * pad - (k - 1) * d
    s = _seed(name)
    x, gy = _randn((B, cin, T), s), _randn((B, cout, t_out), s + 1, 1e-3)
    dw, names = _profiled(lambda: ops.conv1d_wgrad(x.to(dev), gy.to(dev), (cout, cin // G, k), padding=pad, dilation=d,
                                                   groups=G, x_slope=xs, g_slope=gs))
    assert names == ["conv1d_wgrad_tc"], names
    acc, mag, _ = E.conv1d_wgrad_acc(x, gy, k, pad_left=pad, dilation=d, groups=G, x_slope=xs, g_slope=gs)
    ref, beta = E.epilogue_f32(acc, err=E.accumulation_bound(mag, 3 * B * t_out, E.U_TC))
    true = torch.nn.grad.conv1d_weight(F.pad(E.lrelu(x, xs).double(), (pad, pad)), (cout, cin // G, k),
                                       E.lrelu(gy, gs).double(), dilation=d, groups=G)
    _record(name, dw, ref, beta, true)


# ---------------------------------------------------------------------------------------------------- coverage
def check_coverage():
    """The readback tables cover every entry point and loader / epilogue class the issue of rounding reaches (a check
    on the declared tables, no GPU)."""
    tags = set()
    for name, (B, cin, cout, k, d, T, pad, mode, groups, epi, opt, plan) in CONV.items():
        tags.add(f"pad:{mode}")
        tags.add(f"epi:{epi}")
        if pad and pad[0] != pad[1]:
            tags.add("pad:asymmetric")
        if opt.get("off"):
            tags.add("off:x")
        if "post" in opt:
            tags.add("post:lrelu")
        tags.add("loader:" + ("cpasync" if plan.get("tma_act") == 0 else "tma" if plan.get("tma_act") == 1 else "?"))
        tags.add("epilogue:" + ("register" if plan.get("staged") == 0 else "staged"))
        if plan.get("nco", 1) > 1:
            tags.add("nco>1")
        if groups > 1:
            tags.add("grouped")
        if opt.get("special"):
            tags.add("special:" + ("register" if opt.get("variant", 0) & 4 else "staged"))
        scale = opt.get("scale", THIRD)
        tags.add(f"scale:{scale:.4f}")
    required = {"pad:zero", "pad:reflect", "pad:replicate", "pad:asymmetric", "off:x", "post:lrelu", "loader:tma",
                "loader:cpasync", "epilogue:register", "epilogue:staged", "nco>1", "grouped", "special:register",
                "special:staged", f"scale:{THIRD:.4f}", f"scale:{SQRT_HALF:.4f}", "epi:plain", "epi:res", "epi:acc",
                "epi:both"}
    missing = required - tags
    assert not missing, sorted(missing)
    assert sorted(p["staged"] for _, p in TANH.values()) == [0, 1]
    assert {m for *_, m in PAIR.values()} == {"acc", "plain"} and {c for c, *_ in PAIR.values()} == {32, 64}
    assert any(r[2] for r in CONVTR.values()) and any(r[-1]["nco"] > 1 for r in CONVTR.values())
    # every tensor-core readback row names the plan it reads back
    assert all(r[-1] for r in CONVTR.values()) and all(isinstance(r[-1], dict) and r[-1] for r in STRIDED.values())
    assert {r[7] for r in STRIDED.values()} >= {1} and any(r[7] > 1 for r in STRIDED.values())
    assert {r[8] for r in WGRAD.values()} | {r[9] for r in WGRAD.values()} == {0.1, 0.2}
    assert any(o.get("special") for *_, o, _ in FFMA.values()) and {r[6] for r in FFMA.values()} == {"zero", "reflect", "replicate"}
    assert {r[7] for r in FFMA.values()} >= {"both", "res", "plain"}
