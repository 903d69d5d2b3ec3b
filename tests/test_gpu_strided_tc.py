"""Strided discriminator convs on the tensor-core path (space-to-depth + stride-1 tensor-core conv):
forward, data gradient and weight gradient vs torch autograd on the CPU (fp32 oracle of the same op),
at the HiFi-GAN MSD / MPD layer shapes (hifigan.py:354-381, 586-601) and the C5 batch."""
import pytest
import torch
import torch.nn.functional as F

from helpers import max_abs_over_peak, rel_l2
from oracle import synth

pytestmark = pytest.mark.gpu
TC_TOL = 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


CASES = [
    # cin, cout, K, stride, groups, pad, rows, period, B
    (512, 1024, 5, 3, 1, 2, 152, 2, 16),   # MPD p=2 layer 4 at the C5 batch (68 % of the D MACs with the next layer)
    (128, 512, 5, 3, 1, 2, 92, 11, 4),     # MPD p=11 layer 3
    (32, 128, 5, 3, 1, 2, 273, 5, 2),      # MPD layer 2 (cin * s = 96)
    (128, 128, 41, 2, 4, 20, 4096, 1, 4),  # MSD layer 1 (grouped, stride 2)
    (256, 512, 41, 4, 16, 20, 1024, 1, 4),  # MSD layer 3 (cin_g * s = 64)
    (512, 1024, 41, 4, 16, 20, 259, 1, 2),  # MSD layer 4, ragged length
]


@pytest.mark.parametrize("cin,cout,K,stride,groups,pad,rows,P,B", CASES)
def test_strided_conv_s2d_forward_backward(dev, cin, cout, K, stride, groups, pad, rows, P, B):
    from parallelwavegan_b200 import ops

    x = synth.randn((B, cin, rows * P), 1)
    w = synth.randn((cout, cin // groups, K), 2, 1.0 / (cin // groups * K) ** 0.5)
    b = synth.randn((cout,), 3, 0.1)
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    # gradients are compared on the bare conv: with a LeakyReLU epilogue a sign flip of an output within rounding
    # distance of 0 changes that element's gradient by O(1) (a fraction ~1e-5 of the elements -> ~3e-3 rel-L2), which
    # measures the conditioning of the mask, not the kernels; the fused activation is checked on the forward below
    if P == 1:
        ref = F.conv1d(xr, wr, br, stride=stride, padding=pad, groups=groups)
    else:
        ref = F.conv2d(xr.view(B, cin, rows, P), wr.unsqueeze(-1), br, stride=(stride, 1), padding=(pad, 0), groups=groups)
    gy = synth.randn(tuple(ref.shape), 4)
    ref.backward(gy)
    xd, wd, bd = x.to(dev).requires_grad_(True), w.to(dev).requires_grad_(True), b.to(dev).requires_grad_(True)
    xin = xd if P == 1 else xd.view(B, cin, rows, P)
    wq = wd if P == 1 else wd.unsqueeze(-1)
    ops.PROFILE = []
    try:
        y = ops.conv1d(xin, wq, bd, stride=stride, padding=pad, groups=groups, period=P)
        y.backward(gy.to(dev))
        torch.cuda.synchronize()
        names = [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None
    assert "s2d" in names and "conv1d_tc" in names and "conv1d" not in names, names
    assert tuple(y.shape) == tuple(ref.shape)
    assert rel_l2(y.detach().cpu(), ref.detach()) < TC_TOL and max_abs_over_peak(y.detach().cpu(), ref.detach()) < 5 * TC_TOL
    assert rel_l2(xd.grad.cpu(), xr.grad) < TC_TOL
    assert rel_l2(wd.grad.cpu(), wr.grad) < TC_TOL
    assert rel_l2(bd.grad.cpu(), br.grad) < TC_TOL
    # no-grad inference form with the fused LeakyReLU epilogue
    with torch.no_grad():
        y2 = ops.conv1d(xin.detach(), wq.detach(), bd.detach(), stride=stride, padding=pad, groups=groups, period=P, post_act="lrelu", post_slope=0.1)
    assert rel_l2(y2.cpu(), F.leaky_relu(ref.detach(), 0.1)) < TC_TOL


@pytest.mark.parametrize("P,rows,B", [(1, 128, 16), (3, 37, 4)])
def test_logit_conv_on_tensor_cores(dev, P, rows, B):
    """1024 -> 1 logit convs (MSD k3, MPD (3,1)): zero-padded to 16 output channels for the tensor-core path; forward and
    gradients vs torch autograd."""
    from parallelwavegan_b200 import ops

    x = synth.randn((B, 1024, rows * P), 5)
    w = synth.randn((1, 1024, 3), 6, 0.02)
    b = synth.randn((1,), 7, 0.1)
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    if P == 1:
        ref = F.conv1d(xr, wr, br, padding=1)
    else:
        ref = F.conv2d(xr.view(B, 1024, rows, P), wr.unsqueeze(-1), br, padding=(1, 0))
    gy = synth.randn(tuple(ref.shape), 8)
    ref.backward(gy)
    xd, wd, bd = x.to(dev).requires_grad_(True), w.to(dev).requires_grad_(True), b.to(dev).requires_grad_(True)
    ops.PROFILE = []
    try:
        y = ops.conv1d(xd if P == 1 else xd.view(B, 1024, rows, P), wd if P == 1 else wd.unsqueeze(-1), bd, padding=1, period=P)
        y.backward(gy.to(dev))
        torch.cuda.synchronize()
        names = [q[0] for q in ops.PROFILE]
    finally:
        ops.PROFILE = None
    assert names[0] == "conv1d_tc", names  # forward on the tensor cores (the 16-channel-wide gradients stay on FFMA)
    assert tuple(y.shape) == tuple(ref.shape)
    assert rel_l2(y.detach().cpu(), ref.detach()) < TC_TOL
    assert rel_l2(xd.grad.cpu(), xr.grad) < TC_TOL and rel_l2(wd.grad.cpu(), wr.grad) < TC_TOL and rel_l2(bd.grad.cpu(), br.grad) < TC_TOL


def test_conv_transpose_dgrad_on_tensor_cores(dev):
    """Generator upsampler backward (ConvTranspose1d k16 s8): its data gradient is a stride-8 conv -> space-to-depth path."""
    from parallelwavegan_b200 import ops

    x = synth.randn((4, 512, 32), 15)
    w = synth.randn((512, 256, 16), 16, 0.02)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ref = F.conv_transpose1d(F.leaky_relu(xr, 0.1), wr, None, stride=8, padding=4)
    gy = synth.randn(tuple(ref.shape), 17)
    ref.backward(gy)
    xd, wd = x.to(dev).requires_grad_(True), w.to(dev).requires_grad_(True)
    ops.PROFILE = []
    try:
        y = ops.conv_transpose1d(xd, wd, None, stride=8, padding=4, pre_slope=0.1)
        y.backward(gy.to(dev))
        torch.cuda.synchronize()
        names = [q[0] for q in ops.PROFILE]
    finally:
        ops.PROFILE = None
    assert "s2d" in names, names
    assert rel_l2(y.detach().cpu(), ref.detach()) < TC_TOL
    assert rel_l2(wd.grad.cpu(), wr.grad) < TC_TOL
    # the pre-LeakyReLU mask makes a handful of x-gradient elements flip with rounding: compare where |x| is not tiny
    m = x.abs() > 1e-3
    assert rel_l2(xd.grad.cpu()[m], xr.grad[m]) < TC_TOL


def test_grouped_strided_conv_padded_groups_inference(dev):
    """MSD layer 2 (128 -> 256, k41, stride 2, 16 groups): cin_g * s = 16 channels per group after the re-layout, zero-padded
    to 32 for the tensor cores -- used on the no-grad passes only."""
    from parallelwavegan_b200 import ops

    x = synth.randn((4, 128, 2048), 1)
    w = synth.randn((256, 8, 41), 2, 1.0 / (8 * 41) ** 0.5)
    b = synth.randn((256,), 3, 0.1)
    ref = F.leaky_relu(F.conv1d(x, w, b, stride=2, padding=20, groups=16), 0.1)
    ops.PROFILE = []
    try:
        with torch.no_grad():
            y = ops.conv1d(x.to(dev), w.to(dev), b.to(dev), stride=2, padding=20, groups=16, post_act="lrelu", post_slope=0.1)
        torch.cuda.synchronize()
        names = [q[0] for q in ops.PROFILE]
    finally:
        ops.PROFILE = None
    assert names == ["s2d", "conv1d_tc"], names
    assert rel_l2(y.cpu(), ref) < TC_TOL


@pytest.mark.parametrize("mode", ["zero", "reflect"])
def test_mel_input_conv_padded_channels(dev, mode):
    """80 -> 512 k7 input conv (hifigan.py:80-91 / melgan.py:70-72): channels zero-padded to 96 for the tensor-core path;
    forward and gradients vs torch autograd."""
    from parallelwavegan_b200 import ops

    x = synth.randn((3, 80, 200), 21)
    w = synth.randn((512, 80, 7), 22, 1.0 / (80 * 7) ** 0.5)
    b = synth.randn((512,), 23, 0.1)
    xr, wr, br = x.clone().requires_grad_(True), w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    xp = F.pad(xr, (3, 3)) if mode == "zero" else F.pad(xr, (3, 3), mode="reflect")
    ref = F.conv1d(xp, wr, br)
    gy = synth.randn(tuple(ref.shape), 24)
    ref.backward(gy)
    xd, wd, bd = x.to(dev).requires_grad_(True), w.to(dev).requires_grad_(True), b.to(dev).requires_grad_(True)
    ops.PROFILE = []
    try:
        y = ops.conv1d(xd, wd, bd, padding=3, pad_mode=mode)
        y.backward(gy.to(dev))
        torch.cuda.synchronize()
        names = [q[0] for q in ops.PROFILE]
    finally:
        ops.PROFILE = None
    assert names[0] == "conv1d_tc", names
    assert rel_l2(y.detach().cpu(), ref.detach()) < TC_TOL
    assert rel_l2(xd.grad.cpu(), xr.grad) < TC_TOL and rel_l2(wd.grad.cpu(), wr.grad) < TC_TOL and rel_l2(bd.grad.cpu(), br.grad) < TC_TOL
