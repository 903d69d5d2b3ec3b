"""The staged epilogue of the stride-1 tensor-core conv (residual / accumulate through a shared-memory tile and bulk
copies) against the register epilogue it replaces.  The two plans differ only in buffer counts (and MT at 48 and 64
columns), none of which changes the order of the arithmetic, so the outputs must be bit-identical.
pwgb_debug_set(1, 4) forces the register epilogue; pwgb_debug_get(1, ...) reads back the plan of the last launch."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from helpers import max_abs_over_peak, rel_l2

pytestmark = pytest.mark.gpu

TC_TOL = 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _last_plan():
    from parallelwavegan_b200 import capi

    v = (C.c_int * 5)()
    assert capi.lib().pwgb_debug_get(1, C.cast(v, C.c_void_p), C.sizeof(v)) == 0
    return dict(zip(("MT", "na", "nb", "ns", "staged"), list(v)))


def _run(dev, x, w, b, res, prev, k, variant, **kw):
    from parallelwavegan_b200 import capi, ops

    lib = capi.lib()
    lib.pwgb_debug_set(1, variant)
    try:
        out = prev.clone() if prev is not None else None
        y = ops.conv1d(x, w, b, padding=(k - 1) // 2, pre_slope=0.1, residual=res, out=out,
                       accumulate=prev is not None, **kw)
        torch.cuda.synchronize()
        return y, _last_plan()
    finally:
        lib.pwgb_debug_set(1, 0)


def _inputs(dev, B, cin, cout, k, T, mode, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, cin, T, device=dev, generator=g)
    w = torch.randn(cout, cin, k, device=dev, generator=g) / (cin * k) ** 0.5
    b = 0.1 * torch.randn(cout, device=dev, generator=g)
    res = torch.randn(B, cout, T, device=dev, generator=g) if mode in ("res", "both") else None
    prev = torch.randn(B, cout, T, device=dev, generator=g) if mode in ("acc", "both") else None
    return x, w, b, res, prev


@pytest.mark.parametrize(
    "cin,cout,k,T,B,mode",
    [
        (256, 256, 3, 3200, 2, "both"),    # bench stage 0: two column chunks of 128
        (128, 128, 3, 25600, 2, "both"),   # bench stage 1
        (64, 64, 3, 51200, 2, "both"),     # bench stage 2
        (32, 32, 3, 102400, 2, "both"),    # bench stage 3
        (128, 128, 11, 25600, 2, "res"),
        (32, 16, 3, 2052, 2, "both"),      # Cout 16; T = 2052: ragged last tile
        (32, 48, 5, 2052, 2, "both"),      # Cout 48
        (64, 64, 7, 2052, 3, "res"),       # residual only
        (64, 64, 7, 2052, 3, "acc"),       # accumulate only
    ],
)
def test_staged_epilogue_matches_register_epilogue(dev, cin, cout, k, T, B, mode):
    x, w, b, res, prev = _inputs(dev, B, cin, cout, k, T, mode, seed=cin + cout + k + T)
    kw = dict(out_scale=1.0 / 3.0)
    y_st, plan_st = _run(dev, x, w, b, res, prev, k, 0, **kw)
    y_reg, plan_reg = _run(dev, x, w, b, res, prev, k, 4, **kw)
    assert plan_st["staged"] == 1, plan_st
    assert plan_reg["staged"] == 0, plan_reg
    assert torch.equal(y_st, y_reg)


def test_staged_epilogue_post_act(dev):
    """the activation of the epilogue (tanh) runs before the residual, as in the register epilogue"""
    x, w, b, res, prev = _inputs(dev, 2, 32, 32, 3, 2052, "both", seed=11)
    y_st, plan_st = _run(dev, x, w, b, res, prev, 3, 0, post_act="tanh", out_scale=0.5)
    y_reg, _ = _run(dev, x, w, b, res, prev, 3, 4, post_act="tanh", out_scale=0.5)
    assert plan_st["staged"] == 1, plan_st
    assert torch.equal(y_st, y_reg)


def test_ragged_length_keeps_register_epilogue(dev):
    """T_out % 4 != 0: rows are not 16-byte aligned, so the conv falls back to the register epilogue and stays right"""
    B, cin, cout, k, T = 2, 32, 32, 3, 2049
    x, w, b, res, prev = _inputs(dev, B, cin, cout, k, T, "both", seed=7)
    y, plan = _run(dev, x, w, b, res, prev, k, 0, out_scale=0.5)
    assert plan["staged"] == 0, plan
    ref = prev.cpu() + 0.5 * (F.conv1d(F.leaky_relu(x.cpu(), 0.1), w.cpu(), b.cpu(), padding=1) + res.cpu())
    assert rel_l2(y.cpu(), ref) < TC_TOL
    assert max_abs_over_peak(y.cpu(), ref) < TC_TOL * 5


def test_plain_conv_gets_no_staging_tile(dev):
    """a conv with neither residual nor accumulate keeps the register epilogue and its weight stages"""
    x, w, b, _, _ = _inputs(dev, 2, 128, 128, 11, 4096, "none", seed=3)
    _, plan = _run(dev, x, w, b, None, None, 11, 0)
    assert plan["staged"] == 0, plan
