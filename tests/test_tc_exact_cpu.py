"""The exact bf16x3 reference (oracle/bf16x3.py) checked on the CPU, and the case table of tests/test_gpu_tc_exact.py.

The GPU tests compare the tensor-core kernels with this reference by torch.equal, so the reference itself must be right:
- with the dropped lo*lo term added back, the emulation is the fp64 conv of the same fp32 operands, exactly;
- on guarded data, fp32 sums of the terms in any order equal the emulation exactly (the premise of the GPU tests);
- the guard rejects data that break the l = 0 when h = 0 rule;
- ``split`` rounds to nearest even like __floats2bfloat162_rn;
- the GPU case table covers every plan class it is meant to."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bf16x3 as E


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rne_bf16(x):
    """fp32 -> bf16 -> fp32 by integer arithmetic on the bit pattern (round to nearest, ties to even)"""
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return torch.from_numpy(b.astype(np.uint32).view(np.float32))


def test_split_rounds_to_nearest_even():
    ulp = 2.0 ** -7  # bf16 spacing in [1, 2)
    ties = [1 + ulp / 2, 1 + 3 * ulp / 2, -(1 + ulp / 2), -(1 + 3 * ulp / 2), 3 + 2 * ulp / 2, 2 ** -100 * (1 + ulp / 2)]
    x = torch.tensor(ties + [1 + ulp / 2 + 2 ** -20, 1 + ulp / 2 - 2 ** -20], dtype=torch.float32)
    hi, lo = E.split(x)
    expect = torch.tensor([1.0, 1 + 2 * ulp, -1.0, -(1 + 2 * ulp), 3.0, 2.0 ** -100, 1 + ulp, 1.0], dtype=torch.float32)
    assert torch.equal(hi, expect)
    g = torch.Generator().manual_seed(0)
    r = torch.randn(100000, generator=g) * torch.exp2(torch.randint(-30, 30, (100000,), generator=g).float())
    hi, lo = E.split(r)
    assert torch.equal(hi, _rne_bf16(r.numpy()))
    assert torch.equal(lo, _rne_bf16((r - hi).numpy()))


def test_grid_values_split_exactly():
    v = E.grid_values((4096,), _gen(1), scale=2.0 ** -3, hmax=3, zero_frac=0.2)
    hi, lo = E.split(v)
    assert torch.equal(hi + lo, v)
    assert E.grid(hi) >= 2.0 ** -3 and E.grid(lo) >= 2.0 ** -13


def test_grid():
    assert E.grid(torch.tensor([3.0, 0.5, -1.25])) == 0.25
    assert E.grid(torch.tensor([0.0])) == math.inf
    assert E.grid(torch.tensor([2.0 ** -40, 6.0])) == 2.0 ** -40


@pytest.mark.parametrize("pad_mode", ["zero", "reflect", "replicate"])
@pytest.mark.parametrize("groups", [1, 4])
def test_conv1d_emulation_plus_lolo_is_the_fp64_conv(pad_mode, groups):
    """on grid data hi + lo == x, so the four products are the fp64 conv of the fp32 operands, and every fp64 sum is
    exact: equality"""
    g = _gen(2)
    x = E.grid_values((2, 64, 50), g, 1.0, hmax=3)
    w = E.grid_values((32, 64 // groups, 5), g, 2.0 ** -5, hmax=3)
    acc, _, _ = E.conv1d_acc(x, w, padding=(3, 5), dilation=2, groups=groups, pad_mode=pad_mode, pre_slope=0.25, lolo=True)
    a = E.lrelu(x, 0.25).double()
    a = F.pad(a, (3, 5)) if pad_mode == "zero" else F.pad(a, (3, 5), mode=pad_mode)
    assert torch.equal(acc, F.conv1d(a, w.double(), dilation=2, groups=groups))


def test_conv_transpose1d_emulation_plus_lolo_is_the_fp64_conv():
    g = _gen(3)
    x = E.grid_values((2, 64, 20), g, 1.0, hmax=3)
    w = E.grid_values((64, 16, 16), g, 2.0 ** -5, hmax=3)
    y, ex = E.conv_transpose1d(x, w, stride=8, padding=4, pre_slope=0.5)
    xh, xl = E.split(E.lrelu(x, 0.5))
    wh, wl = E.split(w)
    lolo = F.conv_transpose1d(xl.double(), wl.double(), stride=8, padding=4)
    ref = F.conv_transpose1d(E.lrelu(x, 0.5).double(), w.double(), stride=8, padding=4)
    assert ex.ok
    assert torch.equal(y.double() + lolo, ref)


def test_wgrad_emulation_plus_lolo_is_the_fp64_weight_gradient():
    g = _gen(4)
    B, cin, cout, K, D, T = 2, 64, 32, 3, 2, 40
    x = E.grid_values((B, cin, T), g, 1.0, hmax=2)
    gy = E.grid_values((B, cout, T), g, 2.0 ** -4, hmax=2)
    dw, ex = E.conv1d_wgrad(x, gy, K, pad_left=D, dilation=D, x_slope=0.5, g_slope=0.25)
    assert ex.ok
    xr = E.lrelu(x, 0.5).double().requires_grad_(True)
    wr = torch.zeros(cout, cin, K, dtype=torch.float64, requires_grad=True)
    F.conv1d(xr, wr, padding=D, dilation=D).backward(E.lrelu(gy, 0.25).double())
    gh, gl = E.split(E.lrelu(gy, 0.25))
    xh, xl = E.split(E.lrelu(x, 0.5))
    lolo = torch.nn.grad.conv1d_weight(F.pad(xl.double(), (D, D)), (cout, cin, K), gl.double(), dilation=D)
    assert torch.equal(dw.double() + lolo, wr.grad)


def _terms(x, w, pre_slope):
    """every product of the bf16x3 conv (valid padding) as a (terms, outputs) fp32 matrix"""
    xh, xl = E.split(E.lrelu(x, pre_slope))
    wh, wl = E.split(w)
    cols = []
    for a, b in ((xh, wh), (xl, wh), (xh, wl)):
        # (B, cin, T) -> products (B, cout, T_out, cin * K) for k over taps
        u = a.unfold(2, w.shape[2], 1)  # B, cin, T_out, K
        cols.append(torch.einsum("bctk,ock->botck", u.double(), b.double()).reshape(*u.shape[:1], w.shape[0], u.shape[2], -1))
    return torch.cat(cols, dim=-1)  # exact in fp64 (products of two bf16 values)


def test_fp32_sums_in_any_order_equal_the_emulation_on_guarded_data():
    """cin 256, cout 64, k 11, pre-slope 0.5, zero fraction 0.3 (the data of the first guarded run)"""
    g = _gen(5)
    x = E.grid_values((1, 256, 40), g, 1.0, hmax=1, zero_frac=0.3)
    w = E.grid_values((64, 256, 11), g, 2.0 ** -4, hmax=1, zero_frac=0.3)
    y, ex = E.conv1d(x, w, pre_slope=0.5)
    assert ex.ok and ex.bits > 18  # close to the limit, yet exact
    terms = _terms(x, w, 0.5).float()  # every product is exactly fp32
    assert torch.equal(terms.sum(-1, dtype=torch.float64).float(), y)
    seq = torch.zeros(terms.shape[:-1])
    for i in range(terms.shape[-1]):
        seq = seq + terms[..., i]  # fp32, sequential
    assert torch.equal(seq, y)
    perm = torch.randperm(terms.shape[-1], generator=g)
    shuffled = terms[..., perm]
    acc = torch.zeros(terms.shape[:-1])
    for blk in shuffled.split(16, dim=-1):  # fp32 partial sums of 16 products, then a running sum
        acc = acc + blk.sum(-1)
    assert torch.equal(acc, y)


def test_guard_rejects_lo_without_hi():
    """values whose hi part is zero but lo is not put their hi part at the lo scale: the grid collapses and fp32 sums
    stop being exact; the guard must say so (and the same draw with the rule passes)"""
    x_bad = E.grid_values((1, 256, 40), _gen(6), 1.0, hmax=1, zero_frac=0.3, lo_without_hi=True)
    x_good = E.grid_values((1, 256, 40), _gen(6), 1.0, hmax=1, zero_frac=0.3)
    w = E.grid_values((64, 256, 11), _gen(7), 2.0 ** -4, hmax=1, zero_frac=0.3)
    _, ex_bad = E.conv1d(x_bad, w, pre_slope=0.5)
    _, ex_good = E.conv1d(x_good, w, pre_slope=0.5)
    assert ex_good.ok
    assert not ex_bad.ok
    with pytest.raises(AssertionError):
        ex_bad.check()
    # and the sums really are not exact: some fp32 order differs from the fp64 result
    terms = _terms(x_bad, w, 0.5).float()
    exact = terms.sum(-1, dtype=torch.float64)
    seq = torch.zeros(terms.shape[:-1])
    for i in range(terms.shape[-1]):
        seq = seq + terms[..., i]
    assert not torch.equal(seq.double(), exact)


def test_guard_counts_the_epilogue():
    g = _gen(8)
    x = E.grid_values((1, 32, 64), g, 1.0, hmax=3)
    w = E.grid_values((32, 32, 3), g, 2.0 ** -4, hmax=3)
    _, ex = E.conv1d(x, w, padding=1)
    res = torch.full((1, 32, 64), 2.0 ** -30)  # a residual on a finer grid than the conv
    _, ex_res = E.conv1d(x, w, padding=1, residual=res)
    assert ex.ok and not ex_res.ok
    _, ex_scaled = E.conv1d(x, w, padding=1, out_scale=0.5, post_act="lrelu", post_slope=0.5)
    assert ex_scaled.g == ex.g / 4


def test_resblock_pair_emulation_is_two_convs():
    g = _gen(9)
    C, T, k, d = 32, 64, 3, 3
    x = E.grid_values((1, C, T), g, 1.0, hmax=1, lo=False)
    w1 = E.grid_values((C, C, k), g, 2.0 ** -3, hmax=1, lo=False)
    w2 = E.grid_values((C, C, k), g, 2.0 ** -1, hmax=1)
    b1 = E.grid_values((C,), g, 2.0 ** -3, hmax=3, lo=False)
    b2 = E.grid_values((C,), g, 2.0 ** -4, hmax=3)
    y, ex = E.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=0.5, out_scale=0.5)
    assert ex.ok
    h = F.conv1d(E.lrelu(x, 0.5).double(), w1.double(), b1.double(), padding=d, dilation=d)
    assert torch.equal(E.split(h.float())[1], torch.zeros_like(h).float())  # regime (b): h is exactly bf16
    # h_lo = 0, so the dropped h_lo * w2_lo is zero and conv2 is the fp64 conv
    ref = 0.5 * (F.conv1d(E.lrelu(h.float(), 0.5).double(), w2.double(), b2.double(), padding=1) + x.double())
    assert torch.equal(y.double(), ref)


def test_gpu_case_table_covers_every_plan_class():
    import test_gpu_tc_exact as T

    T.check_coverage()
