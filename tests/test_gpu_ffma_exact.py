"""The plain-fp32 (FFMA) kernels bit for bit against the exact fp64 reference (oracle/ffma_exact.py), across their branches.

On grid data every product and partial sum of these kernels is exact in fp32 (the bias gradient and the filter adjoint
carry their long sums in double and round once), so the correct output is unique: each kernel must reproduce the
reference with torch.equal.  That sees a dropped tap, a lost partial chunk, an off-by-one reflect index or a row written
for the wrong group, which the rel-L2 bounds of the other suites let through.  Every case asserts the exactness guard
before it runs the GPU.

Each row names the branch it expects: the FFMA conv and weight gradient are read back (pwgb_debug_get(3) / (4)), the
bias gradient and the filter adjoint, which choose their kernel with a one-line predicate, are mirrored in
``expected_kernel``.  check_coverage() (run on the CPU by tests/test_ffma_exact_cpu.py) checks the tables."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import bf16x3 as E
from oracle import ffma_exact as X
from test_gpu_tc_exact import _assert_equal, _draw, _profiled, _readout

pytestmark = pytest.mark.gpu

SLOPE = 0.5    # pre-activation / gradient slopes: powers of two keep every activated value exact
SCALE = 0.5    # out_scale
PLAN3 = ("kernel", "RCO", "WARPS_CO", "RT", "CI_T", "CO")
PLAN4 = ("path", "narrow_fast", "n", "ci_tiles")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _lib():
    from parallelwavegan_b200 import capi

    return capi.lib()


def _simt():
    """ops with ENGINE = "simt" (restored by the caller)"""
    from parallelwavegan_b200 import ops

    old = ops.ENGINE
    ops.ENGINE = "simt"
    return ops, old


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------------- forward conv
# name: dict(B, cin, cout, K, L, S, D, G, P, pad (left, right), mode, lo ("x" | "w": the operand with lo parts),
#            bias, res, acc, post, plan {PLAN3 fields it must read back})
#   L is the flat input length (t_valid of the period view when P > 1)
def _c(B, cin, cout, K, L, plan, **kw):
    r = dict(B=B, cin=cin, cout=cout, K=K, L=L, S=1, D=1, G=1, P=1, pad=(K // 2, K // 2), mode="zero", lo="x", bias=True,
             res=False, acc=False, post=None, plan=plan)
    r.update(kw)
    return r


G0 = dict(kernel=0)
CONV = {
    # the 12 (RCO, WARPS_CO) x RT instantiations of conv1d_fwd_kernel
    "g88_rt4": _c(2, 16, 64, 3, 700, dict(G0, RCO=8, WARPS_CO=8, RT=4, CI_T=16), res=True, acc=True, post="lrelu"),
    "g88_rt1": _c(2, 8, 64, 3, 40, dict(G0, RCO=8, WARPS_CO=8, RT=1, CI_T=8), lo="w", bias=False),
    "g84_rt4_tt_plus1": _c(2, 24, 40, 5, 1025, dict(G0, RCO=8, WARPS_CO=4, RT=4, CI_T=16), res=True),
    "g84_rt1_asym": _c(3, 8, 32, 3, 78, dict(G0, RCO=8, WARPS_CO=4, RT=1), pad=(2, 0), lo="w", acc=True),
    "g82_groups_tt_minus1": _c(2, 40, 48, 5, 1023, dict(G0, RCO=8, WARPS_CO=2, RT=4, CI_T=16), G=2, post="lrelu"),
    "g82_rt1_dilated": _c(2, 16, 16, 7, 150, dict(G0, RCO=8, WARPS_CO=2, RT=1), D=3, pad=(9, 9), lo="w", res=True, acc=True),
    "g81_cit_halved": _c(1, 16, 8, 41, 8192, dict(G0, RCO=8, WARPS_CO=1, RT=4, CI_T=4), S=4, pad=(20, 20)),
    "g81_rt1_s2": _c(2, 12, 12, 5, 600, dict(G0, RCO=8, WARPS_CO=1, RT=1), S=2, pad=(2, 2), lo="w"),
    "g41_rt4_reflect": _c(2, 8, 5, 3, 2000, dict(G0, RCO=4, WARPS_CO=1, RT=4), mode="reflect"),
    "g41_rt1_replicate": _c(2, 8, 4, 3, 300, dict(G0, RCO=4, WARPS_CO=1, RT=1), mode="replicate", pad=(2, 1), lo="w"),
    "g11_rt4_p5_s3": _c(2, 8, 3, 5, 4998, dict(G0, RCO=1, WARPS_CO=1, RT=4), S=3, P=5, pad=(2, 2)),
    "g11_rt1_p2_s3": _c(2, 4, 1, 5, 399, dict(G0, RCO=1, WARPS_CO=1, RT=1), S=3, P=2, pad=(2, 2), lo="w", post="lrelu"),
    # strides, dilation, periods
    "g_p3_s3": _c(2, 8, 32, 5, 1198, dict(G0, RCO=8, WARPS_CO=4, RT=4), S=3, P=3, pad=(2, 2)),
    "g_s3_d2": _c(2, 16, 16, 7, 1000, dict(G0, RCO=8, WARPS_CO=2, RT=4), S=3, D=2, pad=(6, 6), lo="w", bias=False),
    # conv1d_small_cout_kernel
    "sc_c1": _c(2, 66, 1, 3, 500, dict(kernel=1, CO=1)),
    "sc_c3": _c(2, 100, 3, 5, 333, dict(kernel=1, CO=3), lo="w", post="lrelu"),
    "sc_c4_p3": _c(2, 65, 4, 5, 299, dict(kernel=1, CO=4), S=3, P=3, pad=(2, 2)),
    "sc_c2": _c(1, 128, 2, 3, 1000, dict(kernel=1, CO=2), lo="w", bias=False),
    # conv1d_fewcout_long_kernel (CTAs of 1024 outputs: interior ones and edge ones)
    "fc1_zero": _c(2, 32, 1, 7, 5000, dict(kernel=2, CO=1)),
    "fc2_reflect_1024j": _c(2, 16, 2, 5, 4096, dict(kernel=2, CO=2), mode="reflect", lo="w", post="lrelu"),
    "fc4_c3_replicate": _c(1, 24, 3, 7, 6000, dict(kernel=2, CO=4), mode="replicate"),
    "fc4_s2": _c(2, 8, 4, 8, 10000, dict(kernel=2, CO=4), S=2, pad=(3, 3), lo="w"),
    # recipe layers at their real shapes
    "hifigan_out": _c(2, 32, 1, 7, 102400, dict(kernel=2, CO=1)),
    "hifigan_out_dgrad": _c(2, 1, 32, 7, 102400, dict(G0, RCO=8, WARPS_CO=4, RT=4, CI_T=1), lo="w", bias=False),
    "melgan_out": _c(2, 32, 1, 7, 16384, dict(kernel=2, CO=1), mode="reflect"),
    "mbmelgan_v2_out": _c(2, 48, 4, 7, 8192, dict(kernel=2, CO=4), mode="reflect", lo="w"),
    **{f"mpd_p{P}": _c(2, 1, 32, 5, 8191, dict(G0, RCO=8, WARPS_CO=4, RT=4, CI_T=1), S=3, P=P, pad=(2, 2),
                       lo="w" if P % 2 else "x") for P in (2, 3, 5, 7, 11)},
    "melgand_in": _c(2, 1, 16, 15, 8192, dict(G0, RCO=8, WARPS_CO=2, RT=4, CI_T=1), mode="reflect", lo="w"),
    "melgand_k41_s4_g4": _c(2, 16, 64, 41, 8192, dict(G0, RCO=8, WARPS_CO=2, RT=4, CI_T=4), S=4, G=4, pad=(20, 20),
                            post="lrelu"),
}


def conv_t_out(r):
    t_in = -(-r["L"] // r["P"])
    pl, pr = r["pad"]
    return (t_in + pl + pr - r["D"] * (r["K"] - 1) - 1) // r["S"] + 1


def conv_inputs(r, g, hmax, z):
    B, cin, cout, K, G, P = r["B"], r["cin"], r["cout"], r["K"], r["G"], r["P"]
    oshape = (B, cout, conv_t_out(r)) + ((P,) if P > 1 else ())
    return dict(x=E.grid_values((B, cin, r["L"]), g, 1.0, hmax, z, lo=r["lo"] == "x"),
                w=E.grid_values((cout, cin // G, K), g, 2.0 ** -4, hmax, z, lo=r["lo"] == "w"),
                b=E.grid_values((cout,), g, 2.0 ** -4, 3) if r["bias"] else None,
                res=E.grid_values(oshape, g, 1.0, 3) if r["res"] else None,
                prev=E.grid_values(oshape, g, 2.0, 3) if r["acc"] else None)


def conv_ref(r, d, **over):
    """the reference of row r on inputs d; ``over`` replaces row fields (the CPU test's mutations)"""
    r = dict(r, **over)
    scale = SCALE if (r["res"] or r["acc"]) else 1.0
    return X.conv1d(d["x"], d["w"], d["b"], stride=r["S"], padding=r["pad"], dilation=r["D"], groups=r["G"],
                    pad_mode=r["mode"], period=r["P"], pre_slope=SLOPE, post_act=r["post"], post_slope=0.5,
                    residual=d["res"], out_scale=scale, prev=d["prev"])


def conv_case(name):
    r = CONV[name]

    def make(g, hmax, z):
        d = conv_inputs(r, g, hmax, z)
        return (d,) + conv_ref(r, d)

    return _draw(name, make, r["cin"] // r["G"] * r["K"])


def _run_conv(dev, r, d, post=None):
    ops, old = _simt()
    try:
        prev = d["prev"].to(dev) if d["prev"] is not None else None
        scale = SCALE if (r["res"] or r["acc"]) else 1.0
        with torch.no_grad():
            y, names = _profiled(lambda: ops.conv1d_raw(
                d["x"].to(dev), d["w"].to(dev), d["b"].to(dev) if d["b"] is not None else None, stride=r["S"], padding=r["pad"],
                dilation=r["D"], groups=r["G"], pad_mode=r["mode"], pre_slope=SLOPE, post_act=post or r["post"], post_slope=0.5,
                residual=d["res"].to(dev) if d["res"] is not None else None, out_scale=scale, out=prev,
                accumulate=prev is not None, period=r["P"]))
    finally:
        ops.ENGINE = old
    assert names == ["conv1d"], names
    return y


@pytest.mark.parametrize("name", list(CONV))
def test_conv1d_ffma_exact(dev, name):
    r = CONV[name]
    d, ref, ex = conv_case(name)
    ex.check(name)
    y = _run_conv(dev, r, d)
    got = _readout(3, PLAN3)
    assert {k: got[k] for k in r["plan"]} == r["plan"], got
    _assert_equal(y, ref, name)


# tanh epilogue: on grid data its argument is exact; libdevice's tanhf is within 2 ulp of tanh
@pytest.mark.parametrize("name", ["fc1_zero", "g84_rt4_tt_plus1"])
def test_conv1d_ffma_tanh_within_2ulp(dev, name):
    r = dict(CONV[name], res=False, acc=False, post=None)
    d, z, ex = _draw("tanh_" + name, lambda g, h, zf: (lambda d_: (d_,) + conv_ref(r, d_))(conv_inputs(r, g, h, zf)),
                     r["cin"] * r["K"])
    ex.check(name)
    y = _run_conv(dev, r, d, post="tanh").cpu()
    assert {k: _readout(3, PLAN3)[k] for k in r["plan"]} == r["plan"]
    t = torch.tanh(z.double())
    ulp = torch.from_numpy(np.spacing(t.float().abs().numpy())).double()
    err = (y.double() - t).abs()
    assert bool((err <= 2 * ulp).all()), f"{name}: tanh epilogue {float((err / ulp).max()):.2f} ulp from tanh"


# ---------------------------------------------------------------------------------------------------- conv-transpose
# name: (B, cin, cout, K, stride, padding, output_padding, groups, period, t_in, lo ("x" | "w"), plan)
CONVTR = {
    "ct_groups": (2, 64, 32, 8, 4, 2, 0, 4, 1, 100, "x", dict(G0, RCO=8, WARPS_CO=4, RT=4)),
    "ct_period_op": (2, 16, 8, 5, 3, 2, 1, 1, 3, 60, "w", dict(G0, RCO=8, WARPS_CO=2, RT=4)),
    "ct_cin20": (2, 20, 16, 4, 2, 1, 1, 1, 1, 200, "x", dict(G0, RCO=8, WARPS_CO=4, RT=4)),
}


def convtr_inputs(row, g, hmax, z):
    B, cin, cout, K, s, p, op, G, P, t_in, lo, _ = row
    x = E.grid_values((B, cin, t_in) + ((P,) if P > 1 else ()), g, 1.0, hmax, z, lo=lo == "x")
    return dict(x=x, w=E.grid_values((cin, cout // G, K), g, 2.0 ** -4, hmax, z, lo=lo == "w"),
                b=E.grid_values((cout,), g, 2.0 ** -4, 3))


def convtr_ref(row, d, **over):
    B, cin, cout, K, s, p, op, G, P, t_in, lo, _ = row
    return X.conv_transpose1d(d["x"], d["w"], d["b"], stride=s, padding=over.get("padding", p), output_padding=op, groups=G,
                              period=P, pre_slope=SLOPE)


@pytest.mark.parametrize("name", list(CONVTR))
def test_conv_transpose1d_ffma_exact(dev, name):
    row = CONVTR[name]
    B, cin, cout, K, s, p, op, G, P, t_in, lo, plan = row
    d, ref, ex = _draw(name, lambda g, h, z: (lambda d_: (d_,) + convtr_ref(row, d_))(convtr_inputs(row, g, h, z)),
                       cin // G * math.ceil(K / s))
    ex.check(name)
    ops, old = _simt()
    try:
        with torch.no_grad():
            y, names = _profiled(lambda: ops.conv_transpose1d_raw(d["x"].to(dev), d["w"].to(dev), d["b"].to(dev), stride=s, padding=p,
                                                                  output_padding=op, pre_slope=SLOPE, groups=G, period=P))
    finally:
        ops.ENGINE = old
    assert names == ["conv_transpose1d"], names
    got = _readout(3, PLAN3)
    assert {k: got[k] for k in plan} == plan, got
    _assert_equal(y, ref, name)


# ---------------------------------------------------------------------------------------------------- weight gradient
# name: dict(B, cin, cout, K, L, S, D, G, P, pl, mode, xs, gs, lo ("x" | "g"), acc, plan {PLAN4})
def _w(B, cin, cout, K, L, plan, **kw):
    r = dict(B=B, cin=cin, cout=cout, K=K, L=L, S=1, D=1, G=1, P=1, pl=K // 2, mode="zero", xs=SLOPE, gs=1.0, lo="x", acc=False,
             plan=plan)
    r.update(kw)
    return r


def _tiled(nsplit, ci_tiles):
    return dict(path=0, narrow_fast=0, n=nsplit, ci_tiles=ci_tiles)


def _narrow(fast, blocks):
    return dict(path=1, narrow_fast=fast, n=blocks, ci_tiles=0)


WGRAD = {
    "t_k11_cout40_cin12": _w(2, 12, 40, 11, 1000, _tiled(16, 2)),
    "t_groups_s2_nsplit32": _w(4, 32, 64, 5, 2000, _tiled(32, 1), S=2, G=4, pl=2, gs=SLOPE, lo="g"),
    "t_p3_s3_tvalid": _w(2, 8, 16, 5, 1499, _tiled(8, 1), S=3, P=3, pl=2),
    "t_reflect": _w(2, 16, 32, 7, 600, _tiled(10, 2), mode="reflect", lo="g", gs=SLOPE),
    "t_replicate_many_items": _w(8, 8, 8, 3, 1000, _tiled(32, 1), mode="replicate"),
    "t_acc": _w(2, 16, 16, 3, 300, _tiled(6, 2), acc=True, lo="g"),
    "n_fast_cin1": _w(2, 1, 32, 7, 3000, _narrow(1, 6)),
    "n_general_cout1_s2": _w(2, 16, 1, 4, 4000, _narrow(0, 4), S=2, pl=1, lo="g", gs=SLOPE),
    "n_acc": _w(2, 2, 8, 3, 2100, _narrow(1, 6), acc=True),
    "n_4096": _w(2, 512, 4, 2, 700, _narrow(1, 2), pl=0, lo="g"),
    "n_4097": _w(2, 4097, 1, 1, 300, _tiled(6, 513), pl=0),
    **{f"mpd_p{P}": _w(2, 1, 32, 5, 8191, _narrow(0, 2 * math.ceil(P * ((-(-8191 // P) - 1) // 3 + 1) / 1024)), S=3, P=P, pl=2,
                       lo="g" if P % 2 else "x", xs=1.0) for P in (2, 3, 5, 7, 11)},
}


def wgrad_t_out(r):
    t_in = -(-r["L"] // r["P"])
    return (t_in + 2 * r["pl"] - r["D"] * (r["K"] - 1) - 1) // r["S"] + 1


def wgrad_inputs(r, g, hmax, z):
    B, cin, cout, K, G, P = r["B"], r["cin"], r["cout"], r["K"], r["G"], r["P"]
    gshape = (B, cout, wgrad_t_out(r)) + ((P,) if P > 1 else ())
    return dict(x=E.grid_values((B, cin, r["L"]), g, 1.0, hmax, z, lo=r["lo"] == "x"),
                gy=E.grid_values(gshape, g, 2.0 ** -4, hmax, z, lo=r["lo"] == "g"),
                prev=E.grid_values((cout, cin // G, K), g, 2.0 ** 4, 3) if r["acc"] else None)


def wgrad_ref(r, d, **over):
    r = dict(r, **over)
    return X.conv1d_wgrad(d["x"], d["gy"], r["K"], stride=r["S"], pad_left=r["pl"], dilation=r["D"], groups=r["G"],
                          pad_mode=r["mode"], period=r["P"], x_slope=r["xs"], g_slope=r["gs"], prev=d["prev"])


def wgrad_case(name):
    r = WGRAD[name]
    return _draw(name, lambda g, h, z: (lambda d_: (d_,) + wgrad_ref(r, d_))(wgrad_inputs(r, g, h, z)), r["B"] * wgrad_t_out(r) * r["P"])


def _wgrad_capi(dev, r, x, gy, prev, accumulate):
    """pwgb_conv1d_wgrad through the C ABI (the accumulate flag is not exposed by ops)"""
    from parallelwavegan_b200 import capi, ops

    t_in = -(-r["L"] // r["P"])
    d = capi.Conv1dDesc(batch=r["B"], cin=r["cin"], cout=r["cout"], t_in=t_in, t_out=wgrad_t_out(r), kernel=r["K"], stride=r["S"],
                        dilation=r["D"], groups=r["G"], pad_left=r["pl"], pad_mode=ops._PAD[r["mode"]], period=r["P"], t_valid=r["L"],
                        pre_slope=float(r["xs"]), out_scale=1.0)
    L = _lib()
    nbytes = L.pwgb_conv1d_wgrad_workspace(C.byref(d))
    ws = torch.empty(max(nbytes // 4, 1), device=dev)
    dw = prev.to(dev).clone()
    rc = L.pwgb_conv1d_wgrad(C.byref(d), _p(x), _p(gy), float(r["gs"]), _p(dw), int(accumulate), _p(ws), C.c_size_t(nbytes), _stream())
    capi.check(rc, "pwgb_conv1d_wgrad")
    torch.cuda.synchronize()
    return dw.cpu()


@pytest.mark.parametrize("name", list(WGRAD))
def test_conv1d_wgrad_ffma_exact(dev, name):
    r = WGRAD[name]
    d, ref, ex = wgrad_case(name)
    ex.check(name)
    if r["acc"]:
        dw = _wgrad_capi(dev, r, d["x"].to(dev), d["gy"].to(dev), d["prev"], True)
    else:
        ops, old = _simt()
        try:
            with torch.no_grad():
                dw, names = _profiled(lambda: ops.conv1d_wgrad(d["x"].to(dev), d["gy"].to(dev), (r["cout"], r["cin"] // r["G"], r["K"]),
                                                               stride=r["S"], padding=r["pl"], dilation=r["D"], groups=r["G"],
                                                               pad_mode=r["mode"], x_slope=r["xs"], g_slope=r["gs"], period=r["P"]))
        finally:
            ops.ENGINE = old
        assert names == ["conv1d_wgrad"], names
    assert _readout(4, PLAN4) == r["plan"]
    _assert_equal(dw, ref, name)


@pytest.mark.parametrize("accumulate", [False, True])
def test_conv1d_wgrad_batch0(dev, accumulate):
    """B = 0 launches nothing: dw is zeroed, or kept when accumulating"""
    r = _w(0, 8, 8, 3, 100, None)
    prev = E.grid_values((8, 8, 3), torch.Generator().manual_seed(3), 1.0, 3)
    one = torch.zeros(1, device=dev)
    dw = _wgrad_capi(dev, r, one, one, prev, accumulate)
    _assert_equal(dw, prev if accumulate else torch.zeros_like(prev), "batch0")


# ---------------------------------------------------------------------------------------------------- bias gradient
def expected_kernel(op, *args):
    """The one-line dispatch predicates of pwgb_bias_grad and pwgb_upsample_fir_backward (backward.cu), mirrored:
    bias_grad(B, C, L) -> "small" | "cluster"; fir_df(scale) -> "maxs4" | "maxs8" | "tap"."""
    if op == "bias_grad":
        B, Cc, L = args
        return "small" if B * L < 65536 or Cc >= 592 else "cluster"
    s = args[0]
    return "maxs4" if s <= 4 else ("maxs8" if 2 * s + 1 <= 17 else "tap")


# name: (B, C, L, storage offset in floats, accumulate, lo, expected kernel, cluster path ("vec" | "scalar" | None))
BIAS = {
    "small_short_rows": (2, 64, 1000, 0, False, True, "small", None),
    "small_592_channels": (1, 592, 65536, 0, False, False, "small", None),
    "small_65535": (1, 8, 65535, 0, False, True, "small", None),
    "cluster_65536": (2, 8, 32768, 0, False, False, "cluster", "vec"),
    "cluster_vec": (4, 32, 20000, 0, False, True, "cluster", "vec"),
    "cluster_scalar_l": (4, 16, 20001, 0, False, False, "cluster", "scalar"),
    "cluster_scalar_offset": (4, 16, 20000, 1, False, True, "cluster", "scalar"),
    "cluster_acc": (4, 16, 20000, 0, True, False, "cluster", "vec"),
    "small_acc": (2, 8, 100, 0, True, True, "small", None),
}


def bias_inputs(row, g):
    B, Cc, L, off, acc, lo, _, _ = row
    return dict(g=E.grid_values((B, Cc, L), g, 2.0 ** -3, 3, lo=lo), prev=E.grid_values((Cc,), g, 2.0, 3) if acc else None)


def _bias_grad_capi(dev, g, prev, off):
    from parallelwavegan_b200 import capi

    buf = torch.empty(g.numel() + off, device=dev)
    gd = buf[off:].view(g.shape)
    gd.copy_(g)
    db = (prev if prev is not None else torch.full((g.shape[1],), float("nan"))).to(dev)
    rc = _lib().pwgb_bias_grad(_p(gd), _p(db), g.shape[0], g.shape[1], g.shape[2], int(prev is not None), _stream())
    capi.check(rc, "pwgb_bias_grad")
    torch.cuda.synchronize()
    return db.cpu()


@pytest.mark.parametrize("name", list(BIAS))
def test_bias_grad_exact(dev, name):
    row = BIAS[name]
    B, Cc, L, off, acc, lo, kern, path = row
    assert expected_kernel("bias_grad", B, Cc, L) == kern
    d = bias_inputs(row, torch.Generator().manual_seed(len(name) * 7919))
    ref, ex = X.bias_grad(d["g"], d["prev"])
    ex.check(name)
    _assert_equal(_bias_grad_capi(dev, d["g"], d["prev"], off), ref, name)


# ---------------------------------------------------------------------------------------------------- upsample FIR
# name: (op: "fwd" | "dx" | "df", B, C, T, scale, out_channels (0: C), lo ("x" | "f"))
FIR = {
    "fwd_s4_vec": ("fwd", 2, 3, 100, 4, 0, "x"),
    "fwd_s3_scalar": ("fwd", 2, 3, 101, 3, 0, "f"),
    "fwd_s2_out_channels": ("fwd", 2, 3, 50, 2, 5, "x"),
    "fwd_s5": ("fwd", 1, 2, 77, 5, 0, "f"),
    "fwd_s9": ("fwd", 1, 2, 60, 9, 0, "x"),
    "dx_s4": ("dx", 2, 3, 100, 4, 0, "f"),
    "dx_s3_gy_stride": ("dx", 2, 3, 99, 3, 5, "x"),
    "dx_s9": ("dx", 1, 2, 40, 9, 0, "f"),
    "df_s2": ("df", 2, 4, 300, 2, 0, "x"),
    "df_s4_idle_ranks": ("df", 1, 5, 300, 4, 0, "f"),
    "df_s5_gy_stride": ("df", 2, 3, 200, 5, 4, "x"),
    "df_s3": ("df", 2, 2, 128, 3, 0, "f"),
    "df_s9_tap": ("df", 2, 2, 100, 9, 0, "x"),
    # the PWG conditioning upsampler, scales [4, 4, 4, 4] and the hop-300 recipes' [4, 5, 3, 5], 80 mel channels
    **{f"pwg_{op}_{tag}{i}": (op, 2, 80, 24 * math.prod(sc[:i]), sc[i], 0, "x" if i % 2 else "f")
       for tag, sc in (("a", [4, 4, 4, 4]), ("b", [4, 5, 3, 5])) for i in range(4) for op in ("fwd", "dx", "df")},
}


def fir_inputs(row, g, hmax=3, z=0.0):
    op, B, Cc, T, s, oc, lo = row
    oc = oc or Cc
    # one lo operand per product: fwd x * f, dx gy * f, df gy * x
    f = E.grid_values((2 * s + 1,), g, 2.0 ** -3, 3, lo=lo == "f" and op != "df")
    f[f == 0] = 2.0 ** -3  # every tap nonzero: a dropped tap must show
    x = E.grid_values((B, Cc, T), g, 1.0, hmax, z, lo=lo == "x" and op != "dx")
    gy = E.grid_values((B, oc, T * s), g, 2.0 ** -2, hmax, z, lo=(op, lo) in (("dx", "x"), ("df", "f")))
    return dict(x=x, f=f, gy=gy)


def fir_ref(row, d, **over):
    op, B, Cc, T, s, oc, lo = row
    if op == "fwd":
        return X.upsample_fir(d["x"], over.get("f", d["f"]), s)
    if op == "dx":
        return X.upsample_fir_backward_x(d["gy"][:, :Cc], over.get("f", d["f"]), s)
    return X.upsample_fir_backward_f(d["x"], d["gy"][:, :Cc], s)


def fir_case(name):
    row = FIR[name]
    if row[0] != "df":
        d = fir_inputs(row, torch.Generator().manual_seed(len(name) * 31 + row[4]))
        return (d,) + fir_ref(row, d)
    return _draw(name, lambda g, h, z: (lambda d_: (d_,) + fir_ref(row, d_))(fir_inputs(row, g, h, z)), row[3] * row[4])


@pytest.mark.parametrize("name", list(FIR))
def test_upsample_fir_exact(dev, name):
    from parallelwavegan_b200 import capi, ops

    op, B, Cc, T, s, oc, lo = FIR[name]
    d, ref, ex = fir_case(name)
    ex.check(name)
    x, f, gy = d["x"].to(dev), d["f"].to(dev), d["gy"].to(dev)
    if op == "fwd":
        with torch.no_grad():
            y = ops.upsample_fir(x, f, s, out_channels=oc or None)
        torch.cuda.synchronize()
        if oc:
            assert not y[:, Cc:].any()
            y = y[:, :Cc]
        _assert_equal(y, ref, name)
        return
    gx = torch.full((B, Cc, T), float("nan"), device=dev) if op == "dx" else None
    df = torch.full((2 * s + 1,), float("nan"), device=dev) if op == "df" else None
    rc = _lib().pwgb_upsample_fir_backward(B * Cc, Cc, T, s, _p(x), _p(f), _p(gy), (oc or Cc) * T * s, _p(gx), _p(df), _stream())
    capi.check(rc, "pwgb_upsample_fir_backward")
    torch.cuda.synchronize()
    if op == "df":
        assert expected_kernel("fir_df", s) in ("maxs4", "maxs8", "tap")
    _assert_equal(gx if op == "dx" else df, ref, name)


# ---------------------------------------------------------------------------------------------------- gathers
# name: (op, args...)
GATHER = {
    "s2d_groups_cgo": ("s2d", 2, 16, 4, 50, 1, 2, 3, 27, 32),      # (B, C, groups, rows, P, stride, pad, rows_out, cgo)
    "s2d_period": ("s2d", 2, 8, 1, 40, 3, 3, 2, 15, 0),
    "pad_reflect_t_minus_1": ("pad", 2, 3, 9, 8, 8, "reflect"),   # (B, C, T, left, right, mode)
    "pad_reflect_left_only": ("pad", 2, 3, 20, 5, 0, "reflect"),
    "pad_replicate_right_only": ("pad", 2, 3, 20, 0, 7, "replicate"),
    "pad_replicate_t_minus_1": ("pad", 1, 2, 6, 5, 5, "replicate"),
    "pool_hifigan": ("pool", 2, 3, 101, 4, 2, 2, True),           # (B, C, t_in, k, s, pad, count_include_pad)
    "pool_melgan": ("pool", 2, 3, 101, 4, 2, 1, False),
}


def gather_inputs(row, g):
    op = row[0]
    if op == "s2d":
        _, B, Cc, G, rows, P, s, pad, ro, cgo = row
        return dict(x=E.grid_values((B, Cc, rows, P) if P > 1 else (B, Cc, rows), g, 1.0, 3),
                    gy=E.grid_values((B, G * (cgo or Cc // G * s), ro) + ((P,) if P > 1 else ()), g, 1.0, 3))
    if op == "pad":
        _, B, Cc, T, pl, pr, mode = row
        return dict(x=E.grid_values((B, Cc, T), g, 1.0, 3), gy=E.grid_values((B, Cc, T + pl + pr), g, 1.0, 3))
    _, B, Cc, T, k, s, pad, inc = row
    t_out = (T + 2 * pad - k) // s + 1
    return dict(x=E.grid_values((B, Cc, T), g, 1.0, 3), gy=12.0 * E.grid_values((B, Cc, t_out), g, 1.0, 3))


def gather_ref(row, d, backward):
    op = row[0]
    if op == "s2d":
        _, B, Cc, G, rows, P, s, pad, ro, cgo = row
        return X.s2d_backward(d["gy"], tuple(d["x"].shape), G, s, pad, P, cgo) if backward else X.s2d(d["x"], G, s, pad, ro, P, cgo)
    if op == "pad":
        _, B, Cc, T, pl, pr, mode = row
        return X.pad1d_backward(d["gy"], T, pl, pr, mode) if backward else X.pad1d(d["x"], pl, pr, mode)
    _, B, Cc, T, k, s, pad, inc = row
    return X.avg_pool1d_backward(d["gy"], T, k, s, pad, inc) if backward else X.avg_pool1d(d["x"], k, s, pad, inc)


@pytest.mark.parametrize("backward", [False, True])
@pytest.mark.parametrize("name", list(GATHER))
def test_gather_exact(dev, name, backward):
    from parallelwavegan_b200 import autograd as ag
    from parallelwavegan_b200 import ops

    row = GATHER[name]
    d = gather_inputs(row, torch.Generator().manual_seed(len(name)))
    ref, ex = gather_ref(row, d, backward)
    ex.check(name)
    x, gy = d["x"].to(dev), d["gy"].to(dev)
    op = row[0]
    with torch.no_grad():
        if op == "s2d":
            _, B, Cc, G, rows, P, s, pad, ro, cgo = row
            y = ops.s2d_backward_raw(gy, tuple(x.shape), G, s, pad, P, cgo) if backward else ops.s2d_raw(x, G, s, pad, ro, P, cgo)
        elif op == "pad":
            _, B, Cc, T, pl, pr, mode = row
            y = ops.pad1d_backward(gy, T, pl, pr, mode) if backward else ops.pad1d(x, pl, pr, mode)
        else:
            _, B, Cc, T, k, s, pad, inc = row
            if backward:
                xr = x.clone().requires_grad_(True)
                with torch.enable_grad():
                    ag.AvgPool1dFn.apply(xr, k, s, pad, inc).backward(gy)
                y = xr.grad
            else:
                y = ops.avg_pool1d_raw(x, k, s, pad, inc)
    torch.cuda.synchronize()
    _assert_equal(y, ref, f"{name} {'backward' if backward else 'forward'}")


# ---------------------------------------------------------------------------------------------------- elementwise
def _scaled_sum_capi(dev, xs, a, off):
    from parallelwavegan_b200 import capi

    xd = [X_.to(dev) for X_ in xs]
    if off:
        xd = [torch.empty(X_.numel() + off, device=dev)[off:].copy_(X_.reshape(-1)) for X_ in xs]
    table = torch.tensor([t.data_ptr() for t in xd], dtype=torch.int64, device=dev)
    out = torch.full((xs[0].numel(),), float("nan"), device=dev)
    aligned = all(t.data_ptr() % 16 == 0 for t in xd)
    rc = _lib().pwgb_scaled_sum(_p(table), len(xd), float(a), _p(out), out.numel(), int(aligned), _stream())
    capi.check(rc, "pwgb_scaled_sum")
    torch.cuda.synchronize()
    return out.cpu().view(xs[0].shape)


# name: (n, length, storage offset, lo)
SCALED_SUM = {"vec": (3, 4096, 0, True), "scalar_len": (5, 4097, 0, False), "scalar_offset": (3, 4096, 1, True)}


@pytest.mark.parametrize("name", list(SCALED_SUM))
def test_scaled_sum_exact(dev, name):
    n, length, off, lo = SCALED_SUM[name]
    g = torch.Generator().manual_seed(n * 1000 + length)
    xs = [E.grid_values((length,), g, 1.0, 3, lo=lo) for _ in range(n)]
    ref, ex = X.scaled_sum(xs, 0.125)
    ex.check(name)
    _assert_equal(_scaled_sum_capi(dev, xs, 0.125, off), ref, name)


@pytest.mark.parametrize("b", [0.0, 0.5])
def test_axpby_exact(dev, b):
    """with b = 0 the old y is not read into the result: a y full of NaN must not propagate"""
    from parallelwavegan_b200 import ops

    g = torch.Generator().manual_seed(5)
    x = E.grid_values((3, 1001), g, 1.0, 3)
    y = torch.full_like(x, float("nan")) if b == 0 else E.grid_values((3, 1001), g, 2.0, 3, lo=False)
    ref, ex = X.axpby(0.25, x, b, y)
    ex.check("axpby")
    yd = y.to(dev)
    ops.axpby(0.25, x.to(dev), b, yd)
    torch.cuda.synchronize()
    _assert_equal(yd, ref, f"axpby b={b}")


# name: (mode, lo on "g" | "ref", accumulate)
ACT = {"lrelu": ("lrelu", "g", False), "lrelu_acc": ("lrelu", "g", True), "tanh": ("tanh", "g", False),
       "tanh_ref_lo": ("tanh", "ref", False), "tanh_acc": ("tanh", "g", True), "scale": ("scale", "g", True)}


def act_inputs(row, g):
    mode, lo, acc = row
    gg = E.grid_values((2, 3, 999), g, 2.0 ** -2, 3 if lo == "g" else 1, lo=lo == "g")
    ref = E.grid_values((2, 3, 999), g, 2.0 ** -1 if lo == "ref" else 2.0 ** -2, 1 if lo == "ref" else 3, lo=lo == "ref")
    return dict(g=gg, ref=ref, prev=E.grid_values((2, 3, 999), g, 1.0, 3) if acc else None)


@pytest.mark.parametrize("name", list(ACT))
def test_act_backward_exact(dev, name):
    from parallelwavegan_b200 import ops

    mode, lo, acc = ACT[name]
    d = act_inputs(ACT[name], torch.Generator().manual_seed(len(name)))
    ref, ex = X.act_backward(mode, d["g"], d["ref"], slope=0.125, scale=0.5, prev=d["prev"])
    ex.check(name)
    out = d["prev"].to(dev) if acc else None
    y = ops.act_backward(mode, d["g"].to(dev), d["ref"].to(dev) if mode != "scale" else None, slope=0.125, scale=0.5, out=out,
                         accumulate=acc)
    torch.cuda.synchronize()
    _assert_equal(y, ref, name)


# ---------------------------------------------------------------------------------------------------- MSD layer 2 in training
def test_msd_layer2_autograd_exact(dev):
    """HiFi-GAN MSD layer 2 (128 -> 256, k41, s2, g16, pad 20) with gradients: its 8-channel groups keep forward, data
    gradient (grouped FFMA conv-transpose) and weight gradient on the FFMA kernels"""
    from parallelwavegan_b200 import ops

    B, cin, cout, K, s, G, pad, T = 1, 128, 256, 41, 2, 16, 20, 2048
    t_out = (T + 2 * pad - K) // s + 1
    op = T - ((t_out - 1) * s - 2 * pad + K)

    def make(g, hmax, z):
        x = E.grid_values((B, cin, T), g, 1.0, hmax, z)
        w = E.grid_values((cout, cin // G, K), g, 2.0 ** -4, hmax, z, lo=False)
        b = E.grid_values((cout,), g, 2.0 ** -4, 3)
        gy = E.grid_values((B, cout, t_out), g, 2.0 ** -4, hmax, z, lo=False)
        y, ex = X.conv1d(x, w, b, stride=s, padding=pad, groups=G, pre_slope=SLOPE)
        gxe, ex2 = X.conv_transpose1d(gy, w, None, stride=s, padding=pad, output_padding=op, groups=G)
        gx, ex3 = X.act_backward("lrelu", gxe, x, slope=SLOPE)
        gw, ex4 = X.conv1d_wgrad(x, gy, K, stride=s, pad_left=pad, groups=G, x_slope=SLOPE)
        gb, ex5 = X.bias_grad(gy)
        return x, w, b, gy, (y, gx, gw, gb), ex & ex2 & ex3 & ex4 & ex5

    x, w, b, gy, refs, ex = _draw("msd_layer2", make, B * t_out)
    ex.check("msd_layer2")
    xd, wd, bd = (t.to(dev).requires_grad_(True) for t in (x, w, b))
    with torch.enable_grad():
        (y, names) = _profiled(lambda: ops.conv1d(xd, wd, bd, stride=s, padding=pad, groups=G, pre_slope=SLOPE))
        grads, names_b = _profiled(lambda: torch.autograd.grad(y, (xd, wd, bd), gy.to(dev)))
    assert names == ["conv1d"] and names_b == ["conv1d_wgrad", "conv_transpose1d"], (names, names_b)
    for got, ref, what in zip((y,) + tuple(grads), refs, ("y", "gx", "gw", "gb")):
        _assert_equal(got, ref, "msd_layer2 " + what)


# ---------------------------------------------------------------------------------------------------- determinism
def test_reductions_deterministic(dev):
    """on random (non-grid) data two calls give bit-identical results: the split-reduce weight gradient, both bias
    gradient kernels and the filter adjoint (DESIGN.md section 3.4)"""
    from parallelwavegan_b200 import capi

    g = torch.Generator().manual_seed(11)
    r = WGRAD["t_groups_s2_nsplit32"]
    x = torch.randn(r["B"], r["cin"], r["L"], generator=g).to(dev)
    gy = torch.randn(r["B"], r["cout"], wgrad_t_out(r), generator=g).to(dev)
    prev = torch.zeros(r["cout"], r["cin"] // r["G"], r["K"])
    a, b = (_wgrad_capi(dev, r, x, gy, prev, False) for _ in range(2))
    assert _readout(4, PLAN4)["n"] == 32 and torch.equal(a, b)
    for B, Cc, L in ((2, 8, 1000), (4, 16, 20000)):
        gg = torch.randn(B, Cc, L, generator=g)
        a, b = (_bias_grad_capi(dev, gg, None, 0) for _ in range(2))
        assert torch.equal(a, b), expected_kernel("bias_grad", B, Cc, L)
    for s in (4, 5, 9):
        x = torch.randn(2, 8, 300, generator=g).to(dev)
        gy = torch.randn(2, 8, 300 * s, generator=g).to(dev)
        f = torch.randn(2 * s + 1, generator=g).to(dev)
        out = []
        for _ in range(2):
            df = torch.empty(2 * s + 1, device=dev)
            rc = _lib().pwgb_upsample_fir_backward(16, 8, 300, s, _p(x), _p(f), _p(gy), 0, None, _p(df), _stream())
            capi.check(rc, "pwgb_upsample_fir_backward")
            out.append(df.cpu())
        assert torch.equal(out[0], out[1]), expected_kernel("fir_df", s)


# ---------------------------------------------------------------------------------------------------- coverage
def check_coverage():
    """The tables cover the branches they are meant to pin down (a check on the declared tables, no GPU)."""
    insts, tags = set(), set()
    for name, r in CONV.items():
        p = r["plan"]
        t_out = conv_t_out(r)
        Lout = t_out * r["P"]
        if p["kernel"] == 0:
            insts.add((p["RCO"], p["WARPS_CO"], p["RT"]))
            co_t = p["RCO"] * p["WARPS_CO"]
            cg = r["cout"] // r["G"]
            if cg % co_t:
                tags.add("cout_g%CO_T")
            if r["G"] > 1 and cg > co_t:
                tags.add("groups:tiles_per_group>1")
            if "CI_T" in p and (r["cin"] // r["G"]) % p["CI_T"]:
                tags.add("ragged_ci")
            if p.get("CI_T", 16) < min(16, r["cin"] // r["G"]):
                tags.add("ci_t_halved")
            tt = (8 // p["WARPS_CO"]) * 32 * p["RT"]
            if Lout > tt and min(Lout % tt, tt - Lout % tt) == 1:
                tags.add(f"len:TTj{'+' if Lout % tt == 1 else '-'}1")
            tags.add(f"S{r['S']}")
            if r["D"] > 1:
                tags.add("dilation")
            if r["P"] > 1:
                tags.add(f"P{r['P']}:S{r['S']}")
            tags.add(f"pad:{r['mode']}")
            if r["pad"][0] != r["pad"][1]:
                tags.add("pad:asym")
            tags.add(f"epi:bias{int(r['bias'])}:res{int(r['res'])}:acc{int(r['acc'])}:{r['post']}")
            for k, v in (("res", "residual"), ("acc", "accumulate")):
                if r[k]:
                    tags.add(v)
        elif p["kernel"] == 1:
            assert r["cout"] <= 4 and r["cin"] >= 64 and r["mode"] == "zero" and Lout * r["B"] <= 65536, name
            tags.add(f"small_cout:{r['cout']}")
            if r["cin"] % 8:
                tags.add("small_cout:cin%8")
            if Lout % 32:
                tags.add("small_cout:Lout%32")
            if r["P"] > 1 and r["L"] % r["P"]:
                tags.add("small_cout:t_valid")
        else:
            assert r["cout"] <= 4 and t_out >= 4096 and r["P"] == 1, name
            tags.add(f"fewcout:{p['CO']}:{r['mode']}")
            tags.add(f"fewcout:t_out%1024={int(t_out % 1024 != 0)}")
            if t_out > 2048:
                tags.add("fewcout:interior")
            if r["S"] > 1:
                tags.add("fewcout:stride")
        if r["P"] > 1 and r["L"] % r["P"]:
            tags.add("t_valid")
        tags.add(f"lo:{r['lo']}")
    assert insts == {(a, b, rt) for a, b in ((8, 8), (8, 4), (8, 2), (8, 1), (4, 1), (1, 1)) for rt in (1, 4)}, sorted(insts)
    required = {"cout_g%CO_T", "groups:tiles_per_group>1", "ragged_ci", "ci_t_halved", "len:TTj+1", "len:TTj-1", "S2", "S3", "S4",
                "dilation", "P2:S3", "P3:S3", "P5:S3", "t_valid", "pad:reflect", "pad:replicate", "pad:asym", "residual", "accumulate",
                "small_cout:1", "small_cout:2", "small_cout:3", "small_cout:4", "small_cout:cin%8", "small_cout:Lout%32",
                "small_cout:t_valid", "fewcout:1:zero", "fewcout:2:reflect", "fewcout:4:replicate", "fewcout:t_out%1024=0",
                "fewcout:t_out%1024=1", "fewcout:interior", "fewcout:stride", "lo:x", "lo:w"}
    required |= {"epi:bias1:res1:acc1:lrelu", "epi:bias0:res0:acc0:None", "epi:bias1:res1:acc0:None", "epi:bias1:res0:acc1:None",
                 "epi:bias1:res0:acc0:lrelu", "epi:bias1:res1:acc1:None"}
    missing = required - tags
    assert not missing, sorted(missing)
    # the > 48 KB opt-in: the halved tile of g81_cit_halved (TT 1024, K 41, stride 4, CI_T 4) needs 74 KB
    r = CONV["g81_cit_halved"]
    nr = (1024 - 1) * r["S"] + (r["K"] - 1) * r["D"] + 1
    assert 48 * 1024 < (r["plan"]["CI_T"] * nr + r["plan"]["CI_T"] * r["K"] * 12) * 4 <= 96 * 1024
    # conv-transpose: groups, period, cin % 32, output_padding, outputs dropped at both shuffle edges
    ct = list(CONVTR.values())
    assert any(c[7] > 1 for c in ct) and any(c[8] > 1 for c in ct) and any(c[1] % 32 for c in ct) and any(c[6] for c in ct)

    def drops(c):
        """(outputs dropped at the left shuffle edge, at the right one)"""
        B, cin, cout, K, s, p, op, G, P, t_in, lo, _ = c
        t_out = (t_in - 1) * s - 2 * p + K + op
        return p > 0, ((t_out - 1 + p) // s + 1) * s > t_out + p

    assert any(all(drops(c)) for c in ct)
    # weight gradient: both paths, both narrow loops, the 4096 / 4097 boundary, nsplit below and at 32
    w = WGRAD
    tiled = [r for r in w.values() if r["plan"]["path"] == 0]
    assert any(r["K"] > 8 and r["K"] % 8 for r in tiled) and any((r["cout"] // r["G"]) % 32 for r in tiled)
    assert any((r["cin"] // r["G"]) % 8 for r in tiled) and any(r["G"] > 1 for r in tiled) and any(r["S"] > 1 for r in tiled)
    assert any(r["P"] > 1 and r["L"] % r["P"] for r in tiled) and any(wgrad_t_out(r) * r["P"] % 128 for r in tiled)
    assert {r["mode"] for r in tiled} >= {"reflect", "replicate"} and any(r["gs"] != 1 for r in tiled)
    assert any(r["plan"]["n"] < 32 for r in tiled) and any(r["plan"]["n"] == 32 for r in tiled)
    narrow = [r for r in w.values() if r["plan"]["path"] == 1]
    assert {r["plan"]["narrow_fast"] for r in narrow} == {0, 1}
    assert any(r["cin"] // r["G"] <= 4 for r in narrow) and any(r["cout"] <= 4 for r in narrow)
    assert {r["cout"] * r["cin"] // r["G"] * r["K"] for r in w.values()} >= {4096, 4097}
    assert w["n_4096"]["plan"]["path"] == 1 and w["n_4097"]["plan"]["path"] == 0
    assert any(r["acc"] for r in tiled) and any(r["acc"] for r in narrow)
    for r in w.values():  # the dispatch: narrow for (cin_g <= 4 or cout <= 4) and n <= 4096 and zero padding
        n = r["cout"] * (r["cin"] // r["G"]) * r["K"]
        narrow_ok = (r["cin"] // r["G"] <= 4 or r["cout"] <= 4) and n <= 4096 and r["mode"] == "zero"
        assert r["plan"]["path"] == int(narrow_ok)
        if narrow_ok:
            assert r["plan"]["narrow_fast"] == int(r["P"] == 1 and r["S"] == 1)
            assert r["plan"]["n"] == r["B"] * math.ceil(wgrad_t_out(r) * r["P"] / 1024)
        else:
            assert r["plan"]["n"] == min(32, r["B"] * math.ceil(wgrad_t_out(r) * r["P"] / 128))
            assert r["plan"]["ci_tiles"] == math.ceil(r["cin"] // r["G"] / 8)
    # bias gradient: both kernels, both cluster paths, the 65536 boundary, accumulate on both
    kinds = {(row[6], row[7]) for row in BIAS.values()}
    assert kinds >= {("small", None), ("cluster", "vec"), ("cluster", "scalar")}
    for B, Cc, L, off, acc, lo, kern, path in BIAS.values():
        assert expected_kernel("bias_grad", B, Cc, L) == kern
        if kern == "cluster":
            assert path == ("vec" if L % 4 == 0 and off % 4 == 0 else "scalar")
    assert {B * L for B, _, L, *_ in BIAS.values()} >= {65535, 65536}
    assert any(r[1] >= 592 and r[0] * r[2] >= 65536 for r in BIAS.values()) and {r[6] for r in BIAS.values() if r[4]} == {"small", "cluster"}
    # upsample FIR: forward vector and scalar paths, out_channels > C, scales 2 3 4 5 9, every filter-adjoint kernel
    fir = list(FIR.values())
    assert {r[4] for r in fir if r[0] == "fwd"} >= {2, 3, 4, 5, 9}
    assert any(r[0] == "fwd" and r[4] % 4 == 0 for r in fir) and any(r[0] == "fwd" and r[4] % 4 for r in fir)
    assert any(r[0] == "fwd" and r[5] > r[2] for r in fir)
    assert {expected_kernel("fir_df", r[4]) for r in fir if r[0] == "df"} == {"maxs4", "maxs8", "tap"}
    assert any(r[0] == "df" and r[1] * r[2] < 8 for r in fir) and any(r[0] == "df" and r[5] > r[2] for r in fir)
    assert any(r[0] == "dx" for r in fir)
