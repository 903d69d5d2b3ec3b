"""The tensor-core convolutions bit for bit against the exact bf16x3 reference (oracle/bf16x3.py), across their tile plans.

On grid data (oracle/bf16x3.py) every product and partial sum of the bf16x3 arithmetic is exact in fp32, so the correct
fp32 output is unique whatever the order of accumulation: each kernel must reproduce the fp64 emulation with
torch.equal, at every element.  That sees a wrong tap, row, channel, chunk, halo, padding or residual row, a dropped or
duplicated hi/lo product and a wrong bias or epilogue order, which rel-L2 bounds let through.  Every case asserts the
exactness guard before it runs the GPU.

Every row of the tables names the plan it expects, and the test reads the plan back (ops.PROFILE for the path,
pwgb_debug_get(1 / 2) and ops.resblock_pair_plan for the tile plan), so a planner change that moves a case to another
branch fails here instead of silently losing coverage.  check_coverage() (run on the CPU by tests/test_tc_exact_cpu.py)
checks that the tables cover every plan class."""
import ctypes as C
import math
import zlib

import pytest
import torch

from oracle import bf16x3 as E

pytestmark = pytest.mark.gpu

SLOPE = 0.5  # pre-activation slope: a power of two keeps the bf16 split of the activated values exact
# (hmax, zero fraction) of the grid data, tried in order until the exactness guard passes
LADDER = [(3, 0.0), (2, 0.0), (1, 0.0), (1, 0.4), (1, 0.6), (1, 0.75), (1, 0.85), (1, 0.92), (1, 0.96)]
PLAN1 = ("MT", "na", "nb", "ns", "staged", "tma_act", "win_mode", "nco")
PLAN2 = ("nc", "tg", "ntg", "nsplit")


def _seed(name):
    return zlib.crc32(name.encode())


def _draw(name, make, nterms):
    """make(gen, hmax, zero_frac) -> (..., Exactness) for the first rung of LADDER whose data pass the guard.  Rungs
    whose expected sum of magnitudes (nterms products of 2^10 grid steps each, lrelu halving the grid) is already past
    the limit are skipped."""
    for hmax, z in LADDER:
        mean_h = hmax * (hmax + 1) / (2 * hmax + 1) * (1 - z)
        if nterms * mean_h ** 2 * 2.0 ** 11 > 2.0 ** 21:
            continue
        out = make(torch.Generator().manual_seed(_seed(name)), hmax, z)
        if out[-1].ok:
            return out
    raise AssertionError(f"{name}: no data of the ladder passes the exactness guard")


def _assert_equal(y, ref, what):
    y = y.detach().cpu()
    assert y.shape == ref.shape, (what, tuple(y.shape), tuple(ref.shape))
    if torch.equal(y, ref):
        return
    bad = (y != ref).nonzero()
    d = (y.double() - ref.double()).abs()
    raise AssertionError(f"{what}: {bad.shape[0]} of {ref.numel()} elements differ, first at {bad[:4].tolist()}, "
                         f"max |diff| {float(d.max()):.3e}, peak |ref| {float(ref.abs().max()):.3e}")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _lib():
    from parallelwavegan_b200 import capi

    return capi.lib()


def _readout(key, names):
    v = (C.c_int * len(names))()
    assert _lib().pwgb_debug_get(key, C.cast(v, C.c_void_p), C.sizeof(v)) == 0
    return dict(zip(names, list(v)))


def _profiled(fn):
    from parallelwavegan_b200 import ops

    ops.PROFILE = []
    try:
        y = fn()
        torch.cuda.synchronize()
        return y, [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None


def _at_offset(t, dev, off):
    """a contiguous copy of t on the device whose storage starts `off` floats (4 * off bytes) past a 16-byte boundary"""
    if t is None:
        return None
    buf = torch.empty(t.numel() + off, device=dev)
    v = buf[off:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 4 * off
    return v


# ---------------------------------------------------------------------------------------------------- conv1d_tc
# name: (B, cin, cout, k, d, T, (pad_left, pad_right) or None for "same", pad_mode, groups, epilogue, options, expected plan)
#   epilogue: "plain" | "res" | "acc" | "both" (residual and accumulate)
#   options: variant (pwgb_debug_set(1, v): 2 = cp.async activations, 4 = register epilogue), post ("lrelu": slope 0.5),
#            nobias, off = (x, y, residual) storage offsets in floats
#   plan: the fields of PLAN1 it must read back (None: B = 0, no launch)
CONV = {
    # all 12 (MT, NB16) instantiations
    "mt1_c16": (2, 32, 16, 3, 1, 128, None, "zero", 1, "plain", {}, dict(MT=1, staged=0, tma_act=1, nco=1)),
    "mt1_c32": (2, 32, 32, 3, 1, 128, None, "zero", 1, "both", {}, dict(MT=1, staged=1, tma_act=1, nco=1)),
    "mt1_c48": (2, 32, 48, 3, 1, 100, None, "zero", 1, "res", {}, dict(MT=1, staged=1, tma_act=1)),
    "mt1_c64": (2, 64, 64, 3, 1, 124, None, "zero", 1, "plain", {}, dict(MT=1, staged=0)),
    "mt1_c80": (2, 64, 80, 3, 1, 1028, None, "zero", 1, "acc", {}, dict(MT=1, staged=1)),
    "mt1_c96": (2, 32, 96, 3, 1, 1028, None, "zero", 1, "plain", {}, dict(MT=1, staged=0)),
    "mt1_c112": (2, 64, 112, 3, 1, 1028, None, "zero", 1, "both", {}, dict(MT=1, staged=1)),
    "mt1_c128": (2, 64, 128, 3, 1, 1028, None, "zero", 1, "res", {}, dict(MT=1, staged=1)),
    "mt2_c16": (2, 32, 16, 3, 1, 1028, None, "zero", 1, "both", {}, dict(MT=2, staged=1)),
    "mt2_c32": (2, 32, 32, 3, 1, 1028, None, "zero", 1, "plain", {}, dict(MT=2, staged=0)),
    "mt2_c48": (2, 32, 48, 3, 1, 1028, None, "zero", 1, "plain", {}, dict(MT=2, staged=0)),
    "mt2_c64": (2, 64, 64, 3, 1, 1028, None, "zero", 1, "plain", {}, dict(MT=2, staged=0)),
    # epilogues, staged and forced to the register epilogue
    "epi_plain": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "plain", {}, dict(MT=2, staged=0, tma_act=1)),
    "epi_plain_reg": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "plain", dict(variant=4), dict(MT=2, staged=0)),
    "epi_res": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "res", {}, dict(MT=2, staged=1)),
    "epi_res_reg": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "res", dict(variant=4), dict(MT=2, staged=0)),
    "epi_acc": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "acc", {}, dict(MT=2, staged=1)),
    "epi_acc_reg": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "acc", dict(variant=4), dict(MT=2, staged=0)),
    "epi_both": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "both", {}, dict(MT=2, staged=1)),
    "epi_both_reg": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "both", dict(variant=4), dict(MT=2, staged=0)),
    "epi_lrelu": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "both", dict(post="lrelu"), dict(MT=2, staged=1)),
    "epi_lrelu_reg": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "both", dict(post="lrelu", variant=4), dict(MT=2, staged=0)),
    "epi_nobias": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "res", dict(nobias=True), dict(MT=2, staged=1)),
    "epi_nobias_plain": (2, 32, 64, 5, 1, 2052, None, "zero", 1, "plain", dict(nobias=True, post="lrelu"), dict(MT=2, staged=0)),
    # activation loaders
    "ld_cpasync": (2, 32, 32, 5, 1, 2052, None, "zero", 1, "both", dict(variant=2), dict(MT=2, staged=1, tma_act=0)),
    "ld_reflect": (2, 64, 32, 7, 3, 2052, None, "reflect", 1, "res", {}, dict(MT=2, staged=1, tma_act=0)),
    "ld_replicate": (2, 32, 64, 7, 1, 2052, (5, 1), "replicate", 1, "plain", {}, dict(MT=2, staged=0, tma_act=0)),
    "ld_asym": (2, 32, 32, 5, 2, 2052, (8, 0), "zero", 1, "both", {}, dict(MT=2, staged=1, tma_act=1)),
    "ld_tin_ragged": (2, 32, 32, 3, 1, 2050, (0, 0), "zero", 1, "both", {}, dict(MT=2, staged=1, tma_act=0)),
    "ld_x_off": (2, 32, 32, 3, 1, 2052, None, "zero", 1, "both", dict(off=(1, 0, 0)), dict(MT=2, staged=1, tma_act=0)),
    "ld_y_off": (2, 32, 32, 3, 1, 2052, None, "zero", 1, "both", dict(off=(0, 1, 0)), dict(MT=2, staged=0, tma_act=1)),
    "ld_res_off": (2, 32, 32, 3, 1, 2052, None, "zero", 1, "res", dict(off=(0, 0, 1)), dict(MT=2, staged=0, tma_act=1)),
    "ld_y_off_plain": (2, 32, 48, 3, 1, 2052, None, "zero", 1, "plain", dict(off=(0, 3, 0)), dict(MT=2, staged=0)),
    # tile plans
    "win_mode": (1, 32, 32, 3, 1100, 4100, None, "zero", 1, "both", {}, dict(MT=2, win_mode=1, staged=0, tma_act=0, ns=0)),
    "fallback_c48": (2, 32, 48, 5, 1, 2052, None, "zero", 1, "res", {}, dict(MT=1, staged=1, win_mode=0)),
    "fallback_c64": (2, 64, 64, 5, 1, 2052, None, "zero", 1, "res", {}, dict(MT=1, staged=1, win_mode=0)),
    "chunks_c192": (2, 64, 192, 3, 1, 1028, None, "zero", 1, "res", {}, dict(MT=1, staged=1, nco=2)),
    "chunks_c256": (2, 64, 256, 3, 1, 1028, None, "zero", 1, "acc", {}, dict(MT=1, staged=1, nco=2)),
    "chunks_c256_reg": (1, 64, 256, 3, 1, 1028, None, "zero", 1, "both", dict(variant=4), dict(MT=1, staged=0, nco=2)),
    "groups4": (2, 128, 128, 5, 1, 1028, None, "zero", 4, "res", {}, dict(MT=2, staged=1, nco=4)),
    "groups16": (1, 512, 256, 41, 1, 1024, None, "zero", 16, "acc", {}, dict(MT=2, staged=1, nco=16)),
    "groups16_plain": (1, 512, 256, 41, 1, 1022, None, "zero", 16, "plain", dict(post="lrelu"), dict(MT=2, staged=0, nco=16)),
    # lengths
    "len_1": (2, 32, 32, 3, 1, 1, None, "zero", 1, "both", {}, dict(MT=1, staged=0, tma_act=0)),
    "len_4": (2, 32, 32, 3, 1, 4, None, "zero", 1, "both", {}, dict(MT=1, staged=1, tma_act=1)),
    "len_below_halo": (2, 32, 32, 11, 5, 20, None, "zero", 1, "res", {}, dict(MT=1, staged=1, tma_act=1)),
    "len_1020": (2, 32, 32, 3, 1, 1020, None, "zero", 1, "both", {}, dict(MT=2, staged=1)),
    "len_1023": (2, 32, 32, 3, 1, 1023, None, "zero", 1, "both", {}, dict(MT=2, staged=0, tma_act=0)),
    "len_1025": (2, 32, 32, 3, 1, 1025, None, "zero", 1, "both", {}, dict(MT=2, staged=0, tma_act=0)),
    "len_1028": (2, 32, 32, 3, 1, 1028, None, "zero", 1, "both", {}, dict(MT=2, staged=1)),
    "len_127": (2, 64, 96, 3, 1, 127, None, "zero", 1, "both", {}, dict(MT=1, staged=0)),
    "len_132": (2, 64, 96, 3, 1, 132, None, "zero", 1, "both", {}, dict(MT=1, staged=1)),
    "batch_0": (0, 32, 32, 3, 1, 1028, None, "zero", 1, "both", {}, None),  # an empty result, no launch
    # more than 3 x 132 tiles, total % grid != 0: ring counters and the RES_FULL parity wrap
    "many_tiles_mt2": (2, 32, 32, 3, 1, 256 * 250 + 4, None, "zero", 1, "both", {}, dict(MT=2, staged=1)),
    "many_tiles_mt1": (2, 64, 64, 3, 1, 128 * 200 + 4, None, "zero", 1, "res", {}, dict(MT=1, staged=1)),
}


def _conv_case(name):
    B, cin, cout, k, d, T, pad, pad_mode, groups, epi, opt, plan = CONV[name]
    pad = pad or ((k - 1) // 2 * d, (k - 1) // 2 * d)
    t_out = T + pad[0] + pad[1] - (k - 1) * d
    post = opt.get("post")

    def make(g, hmax, z):
        x = E.grid_values((B, cin, T), g, 1.0, hmax, z)
        w = E.grid_values((cout, cin // groups, k), g, 2.0 ** -4, hmax, z)
        b = None if opt.get("nobias") else E.grid_values((cout,), g, 2.0 ** -4, 3)
        res = E.grid_values((B, cout, t_out), g, 1.0, 3) if epi in ("res", "both") else None
        prev = E.grid_values((B, cout, t_out), g, 2.0, 3) if epi in ("acc", "both") else None
        ref, ex = E.conv1d(x, w, b, padding=pad, dilation=d, groups=groups, pad_mode=pad_mode, pre_slope=SLOPE, post_act=post,
                           post_slope=0.5, residual=res, out_scale=0.5, prev=prev)
        return x, w, b, res, prev, ref, ex

    return _draw(name, make, cin // groups * k), (B, cout, t_out, pad, pad_mode, d, groups, epi, opt, plan)


@pytest.mark.parametrize("name", list(CONV))
def test_conv1d_tc_exact(dev, name):
    from parallelwavegan_b200 import ops

    (x, w, b, res, prev, ref, ex), (B, cout, t_out, pad, pad_mode, d, groups, epi, opt, plan) = _conv_case(name)
    ex.check(name)
    ox, oy, orr = opt.get("off", (0, 0, 0))
    xd, resd = _at_offset(x, dev, ox), _at_offset(res, dev, orr)
    out = None
    if prev is not None:
        out = _at_offset(prev, dev, oy)
    elif oy:
        out = _at_offset(torch.zeros(B, cout, t_out), dev, oy)
    lib = _lib()
    lib.pwgb_debug_set(1, opt.get("variant", 0))
    try:
        with torch.no_grad():
            y, names = _profiled(lambda: ops.conv1d(xd, w.to(dev), b.to(dev) if b is not None else None, padding=pad, dilation=d,
                                                    groups=groups, pad_mode=pad_mode, pre_slope=SLOPE, post_act=opt.get("post"),
                                                    post_slope=0.5, residual=resd, out_scale=0.5, out=out,
                                                    accumulate=prev is not None))
        got = _readout(1, PLAN1)
    finally:
        lib.pwgb_debug_set(1, 0)
    assert names == (["conv1d_tc"] if B else []), names  # an empty batch launches nothing
    if out is not None:
        assert y is out
    if plan is not None:
        assert {k: got[k] for k in plan} == plan, got
    _assert_equal(y, ref, name)


# ---------------------------------------------------------------------------------------------------- fused ResBlock pair
PAIR_VARIANTS = [(C, k, d) for C in (32, 64) for k in (3, 7, 11) for d in (1, 3, 5)]


def _pair_case(name, B, C, T, k, d, mode, regime):
    """regime "a": w2 exactly bf16 (the h_lo path); "b": x, w1 and b1 exactly bf16, so h has no lo part (the w2_lo path)"""

    def make(g, hmax, z):
        x = E.grid_values((B, C, T), g, 1.0, hmax, z, lo=regime != "b")
        # the weights' scales keep the residual x within 2^18 steps of conv2's grid
        w1 = E.grid_values((C, C, k), g, 2.0 ** -3, hmax, z, lo=regime != "b")
        b1 = E.grid_values((C,), g, 2.0 ** -3, 3, lo=regime != "b")
        w2 = E.grid_values((C, C, k), g, 2.0 ** -1, hmax, z, lo=regime != "a")
        b2 = E.grid_values((C,), g, 2.0 ** -1, 3)
        prev = E.grid_values((B, C, T), g, 2.0, 3) if mode == "acc" else None
        ref, ex = E.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=SLOPE, out_scale=0.5, prev=prev)
        return x, w1, b1, w2, b2, prev, ref, ex

    return _draw(name, make, 4 * C * k)


def _run_pair(dev, name, B, C, T, k, d, mode, regime):
    from parallelwavegan_b200 import ops

    x, w1, b1, w2, b2, prev, ref, ex = _pair_case(name, B, C, T, k, d, mode, regime)
    ex.check(name)
    plan = ops.resblock_pair_plan(C, T, k, d, batch=B)
    assert plan is not None and plan["TT"] == (256 if C == 32 else 128), plan
    out = None
    if mode == "acc":
        out = prev.to(dev)
    elif mode == "out":
        out = torch.full((B, C, T), float("nan"), device=dev)
    with torch.no_grad():
        y, names = _profiled(lambda: ops.resblock_pair(x.to(dev), w1.to(dev), b1.to(dev), w2.to(dev), b2.to(dev), kernel_size=k,
                                                       dilation=d, slope=SLOPE, out=out, accumulate=mode == "acc",
                                                       out_scale=0.5))
    assert names == ["resblock_pair_tc"], names
    if out is not None:
        assert y is out
    _assert_equal(y, ref, name)


@pytest.mark.parametrize("regime", ["a", "b"])
@pytest.mark.parametrize("mode", ["plain", "out", "acc"])
@pytest.mark.parametrize("C,k,d", PAIR_VARIANTS)
def test_resblock_pair_exact(dev, C, k, d, mode, regime):
    _run_pair(dev, f"pair_{C}_{k}_{d}_{mode}_{regime}", 1, C, 1028, k, d, mode, regime)


# name: (B, C, T, k, d, mode, regime)
PAIR_EXTRA = {
    "below_halo": (2, 32, 8, 11, 5, "acc", "a"),
    "below_halo_c64": (2, 64, 12, 7, 5, "out", "b"),
    "ragged_mt1": (2, 64, 1000, 11, 3, "acc", "b"),
    # several tiles per CTA; more than 3 x 132 tiles and a partial last round at MT = 2
    "many_tiles_mt2": (2, 32, 50000, 11, 5, "acc", "a"),
    "many_tiles_mt1": (2, 64, 16000, 3, 1, "out", "b"),
}


@pytest.mark.parametrize("name", list(PAIR_EXTRA))
def test_resblock_pair_exact_lengths(dev, name):
    _run_pair(dev, "pair_" + name, *PAIR_EXTRA[name])


# ---------------------------------------------------------------------------------------------------- conv_transpose1d
# HiFi-GAN v1 upsamplers: (B, cin, cout, k, stride, padding, t_in) -> column chunks of the virtual (cout * stride) conv
CONVTR = {
    "up0_512_256_k16s8": (1, 512, 256, 16, 8, 4, 32, dict(MT=1, nco=16)),
    "up1_256_128_k16s8": (1, 256, 128, 16, 8, 4, 64, dict(MT=1, nco=8)),
    "up2_128_64_k4s2": (1, 128, 64, 4, 2, 1, 512, dict(MT=1, nco=1)),
    "up3_64_32_k4s2": (2, 64, 32, 4, 2, 1, 1024, dict(MT=2, nco=1)),
    "up_batch_0": (0, 64, 32, 4, 2, 1, 1024, None),
}


@pytest.mark.parametrize("name", list(CONVTR))
def test_conv_transpose1d_tc_exact(dev, name):
    from parallelwavegan_b200 import ops

    B, cin, cout, k, s, p, t_in, plan = CONVTR[name]

    def make(g, hmax, z):
        x = E.grid_values((B, cin, t_in), g, 1.0, hmax, z)
        w = E.grid_values((cin, cout, k), g, 2.0 ** -4, hmax, z)
        b = E.grid_values((cout,), g, 2.0 ** -4, 3)
        return (x, w, b) + E.conv_transpose1d(x, w, b, stride=s, padding=p, pre_slope=SLOPE)

    x, w, b, ref, ex = _draw(name, make, cin * math.ceil(k / s))
    ex.check(name)
    with torch.no_grad():
        y, names = _profiled(lambda: ops.conv_transpose1d(x.to(dev), w.to(dev), b.to(dev), stride=s, padding=p, pre_slope=SLOPE))
    assert names == (["conv_transpose1d"] if B else []), names
    if plan is not None:
        got = _readout(1, PLAN1)
        assert {k_: got[k_] for k_ in plan} == plan, got
    _assert_equal(y, ref, name)


# ---------------------------------------------------------------------------------------------------- strided convs
# the discriminator layers of tests/test_gpu_strided_tc.py (space-to-depth + stride-1 tensor-core conv), smaller batches:
# (cin, cout, K, stride, groups, pad, rows, period, B, post_act)
STRIDED = {
    "mpd_p2_l4": (512, 1024, 5, 3, 1, 2, 152, 2, 1, None),
    "mpd_p11_l3": (128, 512, 5, 3, 1, 2, 92, 11, 1, "lrelu"),
    "mpd_l2": (32, 128, 5, 3, 1, 2, 273, 5, 2, "lrelu"),
    "msd_l1": (128, 128, 41, 2, 4, 20, 4096, 1, 1, "lrelu"),
    "msd_l2_padded_groups": (128, 256, 41, 2, 16, 20, 2048, 1, 1, "lrelu"),
    "msd_l3": (256, 512, 41, 4, 16, 20, 1024, 1, 2, None),
    "msd_l4_ragged": (512, 1024, 41, 4, 16, 20, 259, 1, 2, "lrelu"),
}


@pytest.mark.parametrize("name", list(STRIDED))
def test_strided_conv_tc_exact(dev, name):
    from parallelwavegan_b200 import ops

    cin, cout, K, s, G, pad, rows, P, B, post = STRIDED[name]

    def make(g, hmax, z):
        x = E.grid_values((B, cin, rows * P), g, 1.0, hmax, z)
        w = E.grid_values((cout, cin // G, K), g, 2.0 ** -4, hmax, z)
        b = E.grid_values((cout,), g, 2.0 ** -4, 3)
        # a (K, 1) conv2d over the (rows, P) view is a 1-D conv of every column p
        xc = x.view(B, cin, rows, P).permute(0, 3, 1, 2).reshape(B * P, cin, rows)
        ref, ex = E.conv1d(xc, w, b, stride=s, padding=pad, groups=G, pre_slope=1.0, post_act=post, post_slope=0.5)
        ref = ref.view(B, P, cout, -1).permute(0, 2, 3, 1)
        return x, w, b, (ref if P > 1 else ref[..., 0]).contiguous(), ex

    x, w, b, ref, ex = _draw(name, make, cin // G * K)
    ex.check(name)
    xd = x.to(dev) if P == 1 else x.to(dev).view(B, cin, rows, P)
    wd = w.to(dev) if P == 1 else w.to(dev).unsqueeze(-1)
    with torch.no_grad():
        y, names = _profiled(lambda: ops.conv1d(xd, wd, b.to(dev), stride=s, padding=pad, groups=G, period=P, post_act=post,
                                                post_slope=0.5))
    assert names == ["s2d", "conv1d_tc"], names
    _assert_equal(y, ref, name)


# ---------------------------------------------------------------------------------------------------- weight gradient
# name: (B, cin, cout, k, d, pad, T, groups, x_slope, g_slope, expected {nc, tg, ntg, nsplit}, vec_a, vec_b)
#   vec_a: 16-byte gradient loads (T_out % 4 == 0); vec_b: 16-byte activation loads (T_in, the window rows and
#   k0 * d - pad all multiples of 4) -- the wgrad kernel decides both itself, the table records which one a case runs
WGRAD = {
    "nc64_k1": (2, 64, 64, 1, 1, 0, 1024, 1, 0.5, 1.0, dict(nc=64, tg=1, ntg=1, nsplit=2), True, True),
    "nc64_k2": (1, 128, 64, 2, 1, 0, 512, 1, 1.0, 0.5, dict(nc=64, tg=2, ntg=1, nsplit=1), False, False),
    "ntg3_k11": (2, 32, 64, 11, 1, 5, 1024, 1, 0.5, 1.0, dict(nc=32, tg=4, ntg=3, nsplit=2), True, False),
    "cout40": (2, 32, 40, 3, 2, 0, 1028, 1, 0.5, 1.0, dict(nc=32, tg=3, ntg=1, nsplit=2), True, True),
    "cout160": (2, 64, 160, 3, 1, 1, 1024, 1, 0.5, 0.5, dict(nc=32, tg=3, ntg=1, nsplit=2), True, False),
    "groups4": (2, 128, 128, 5, 1, 2, 1024, 4, 0.5, 1.0, dict(nc=32, tg=4, ntg=2, nsplit=2), True, False),
    "nsplit16": (4, 32, 64, 3, 2, 0, 4100, 1, 0.5, 1.0, dict(nc=32, tg=3, ntg=1, nsplit=16), True, True),
    "tout_ragged": (2, 32, 32, 3, 1, 1, 1023, 1, 0.5, 1.0, dict(nc=32, tg=3, ntg=1, nsplit=2), False, False),
}


@pytest.mark.parametrize("name", list(WGRAD))
def test_conv1d_wgrad_tc_exact(dev, name):
    from parallelwavegan_b200 import ops

    B, cin, cout, k, d, pad, T, G, xs, gs, plan, _, _ = WGRAD[name]
    t_out = T + 2 * pad - (k - 1) * d

    def make(g, hmax, z):
        x = E.grid_values((B, cin, T), g, 1.0, hmax, z)
        gy = E.grid_values((B, cout, t_out), g, 2.0 ** -4, hmax, z)
        return (x, gy) + E.conv1d_wgrad(x, gy, k, pad_left=pad, dilation=d, groups=G, x_slope=xs, g_slope=gs)

    x, gy, ref, ex = _draw(name, make, B * t_out)
    ex.check(name)
    with torch.no_grad():
        dw, names = _profiled(lambda: ops.conv1d_wgrad(x.to(dev), gy.to(dev), (cout, cin // G, k), padding=pad, dilation=d, groups=G,
                                                       x_slope=xs, g_slope=gs))
    assert names == ["conv1d_wgrad_tc"], names
    got = _readout(2, PLAN2)
    assert got == plan, got
    _assert_equal(dw, ref, name)


# ---------------------------------------------------------------------------------------------------- coverage
def check_coverage():
    """The tables cover every plan class the tests are meant to pin down (a check on the declared tables, no GPU)."""
    insts = set()
    tags = set()
    for name, (B, cin, cout, k, d, T, pad, pad_mode, groups, epi, opt, plan) in CONV.items():
        if plan is None:
            tags.add("B=0")
            continue
        cout_g = cout // groups
        chunk = cout_g if cout_g <= 128 else max(c for c in range(16, 129, 16) if cout_g % c == 0)
        insts.add((plan["MT"], chunk // 16))
        staged = plan.get("staged")
        reg = "reg" if opt.get("variant", 0) & 4 else ("staged" if staged else "other")
        tags.add(f"epi:{epi}:{reg}")
        if opt.get("post") == "lrelu":
            tags.add("post:lrelu")
        if opt.get("nobias"):
            tags.add("nobias")
        if opt.get("variant", 0) & 2:
            tags.add("loader:cpasync_forced")
        if plan.get("tma_act") == 1:
            tags.add("loader:tma")
        tags.add(f"pad:{pad_mode}")
        if pad and pad[0] != pad[1]:
            tags.add("pad:asymmetric")
        if T % 4:
            tags.add("t_in%4")
        off = opt.get("off", (0, 0, 0))
        for i, what in enumerate(("x", "y", "res")):
            if off[i]:
                tags.add(f"off:{what}")
                assert what == "x" or plan.get("staged") == 0, name  # a misaligned y / residual turns staging off
        if plan.get("win_mode") == 1:
            tags.add("win_mode")
            assert (k - 1) * d > 2048, name
        if plan.get("MT") == 1 and plan.get("staged") == 1 and cout in (48, 64) and T > 128 and epi in ("res", "both"):
            tags.add(f"fallback:{cout}")
        if plan.get("nco", 1) > 1 and groups == 1:
            tags.add(f"chunks:{cout}:{epi}")
        if groups > 1:
            tags.add(f"groups:{groups}")
        if T in (1, 4):
            tags.add(f"T={T}")
        if T < (k - 1) * d:
            tags.add("T<halo")
        tt = 128 * plan["MT"]
        if T > tt and min(T % tt, tt - T % tt) in (1, 4):
            tags.add(f"T=128MTj{'+' if T % tt < tt // 2 else '-'}{min(T % tt, tt - T % tt)}")
        tiles = B * math.ceil(T / tt)
        if tiles > 3 * 132 and tiles % 132 and epi in ("res", "both"):
            tags.add(f"many_tiles:MT{plan['MT']}")
    assert insts == {(1, n) for n in range(1, 9)} | {(2, n) for n in range(1, 5)}, sorted(insts)
    required = {f"epi:{e}:{p}" for e in ("res", "acc", "both") for p in ("staged", "reg")} | {"epi:plain:other", "epi:plain:reg"}
    required |= {"post:lrelu", "nobias", "loader:tma", "loader:cpasync_forced", "pad:reflect", "pad:replicate", "pad:asymmetric",
                 "t_in%4", "off:x", "off:y", "off:res", "win_mode", "fallback:48", "fallback:64", "groups:4", "groups:16",
                 "T=1", "T=4", "T<halo", "T=128MTj+1", "T=128MTj-1", "T=128MTj+4", "T=128MTj-4", "B=0",
                 "many_tiles:MT1", "many_tiles:MT2"}
    required |= {"chunks:192:res", "chunks:256:acc"}
    missing = required - tags
    assert not missing, sorted(missing)
    # the fused pair: every v1 (C, k, d), both data regimes, plain / out / accumulate (parametrized), and the lengths
    assert sorted(PAIR_VARIANTS) == sorted((C, k, d) for C in (32, 64) for k in (3, 7, 11) for d in (1, 3, 5))
    assert any(T < (k - 1) * d for (_, _, T, k, d, _, _) in PAIR_EXTRA.values())
    # several tiles per CTA (more than 132 tiles of M2 output rows) at both tile heights
    assert {C for (B, C, T, k, _, _, _) in PAIR_EXTRA.values() if B * math.ceil(T / ((128 * (2 if C == 32 else 1) - (k - 1)) & ~3)) > 132} == {32, 64}
    # conv-transpose: the four v1 upsamplers, one of them in 16 column chunks
    assert max(p["nco"] for *_, p in CONVTR.values() if p) == 16
    # weight gradient: every plan branch and both load widths
    w = list(WGRAD.values())
    assert any(r[10]["nc"] == 64 for r in w) and any(r[10]["ntg"] > 1 for r in w) and any(r[10]["nsplit"] > 1 for r in w)
    assert any(r[2] // r[7] % 128 and r[2] // r[7] < 128 for r in w) and any(r[2] // r[7] > 128 and r[2] // r[7] % 128 for r in w)
    assert any(r[7] > 1 for r in w)
    assert {r[11] for r in w} == {True, False} and {r[12] for r in w} == {True, False}
    for B, cin, cout, k, d, pad, T, G, *_, vec_a, vec_b in w:
        t_out = T + 2 * pad - (k - 1) * d
        tg = min(k, 128 // (64 if (cin // G) % 64 == 0 and k <= 2 else 32))
        assert vec_a == (t_out % 4 == 0)
        assert vec_b == (T % 4 == 0 and (128 + (tg - 1) * d) % 4 == 0 and all((k0 * d - pad) % 4 == 0 for k0 in range(0, k, tg)))
