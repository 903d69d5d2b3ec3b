"""The fused ResBlock conv pair (csrc/resblock_tc.cu) against the two tensor-core conv launches it replaces.  The fused
kernel uses the same weight images, bf16x3 split and MMA order into every accumulator, and the same epilogue order, so
the outputs must be bit-identical.  ops.PROFILE shows which path ran."""
import pytest
import torch

from helpers import max_abs_over_peak, rel_l2

pytestmark = pytest.mark.gpu

SLOPE = 0.1


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _inputs(dev, B, C, T, k, seed, bias=True):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, C, T, device=dev, generator=g)
    w1 = torch.randn(C, C, k, device=dev, generator=g) / (C * k) ** 0.5
    w2 = torch.randn(C, C, k, device=dev, generator=g) / (C * k) ** 0.5
    b1 = 0.1 * torch.randn(C, device=dev, generator=g) if bias else None
    b2 = 0.1 * torch.randn(C, device=dev, generator=g) if bias else None
    return x, w1, b1, w2, b2


def _profiled(fn):
    from parallelwavegan_b200 import ops

    ops.PROFILE = []
    try:
        y = fn()
        torch.cuda.synchronize()
        return y, [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None


def _two_launches(x, w1, b1, w2, b2, k, d, out=None, accumulate=False, out_scale=1.0):
    from parallelwavegan_b200 import ops

    xt = ops.conv1d(x, w1, b1, dilation=d, padding=(k - 1) // 2 * d, pre_slope=SLOPE)
    return ops.conv1d(xt, w2, b2, padding=(k - 1) // 2, pre_slope=SLOPE, residual=x, out=out, accumulate=accumulate,
                      out_scale=out_scale)


def _check(dev, B, C, T, k, d, mode="plain", seed=0, bias=True):
    from parallelwavegan_b200 import ops

    x, w1, b1, w2, b2 = _inputs(dev, B, C, T, k, seed, bias)
    kw = {}
    prev = None
    if mode != "plain":  # last pair of a block: out (+)= x' / 3
        prev = torch.randn(B, C, T, device=dev, generator=torch.Generator(device=dev).manual_seed(seed + 1))
        kw = dict(out_scale=1.0 / 3.0, accumulate=mode == "acc")
    with torch.no_grad():
        out_f = prev.clone() if prev is not None else None
        y_f, names = _profiled(lambda: ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=SLOPE, out=out_f, **kw))
        out_r = prev.clone() if prev is not None else None
        y_r, names_r = _profiled(lambda: _two_launches(x, w1, b1, w2, b2, k, d, out=out_r, **kw))
    assert names == ["resblock_pair_tc"], names
    assert names_r == ["conv1d_tc", "conv1d_tc"], names_r
    if prev is not None:
        assert y_f is out_f
    assert torch.equal(y_f, y_r)


@pytest.mark.parametrize("C", [32, 64])
@pytest.mark.parametrize("k", [3, 7, 11])
@pytest.mark.parametrize("d", [1, 3, 5])
def test_v1_pairs_bit_identical(dev, C, k, d):
    # T = 2052: not a multiple of any tile's output rows (124 / 120 / 116)
    _check(dev, 2, C, 2052, k, d, seed=C + k + d)


@pytest.mark.parametrize("C,k,d", [(32, 11, 5), (64, 11, 5), (32, 3, 1)])
@pytest.mark.parametrize("T", [4, 8, 48])
def test_shorter_than_halo(dev, C, k, d, T):
    _check(dev, 3, C, T, k, d, seed=T)


@pytest.mark.parametrize("C,k,d", [(32, 7, 5), (64, 11, 3)])
@pytest.mark.parametrize("mode", ["out", "acc"])
def test_last_pair_writes_out(dev, C, k, d, mode):
    _check(dev, 2, C, 4100, k, d, mode=mode, seed=5)


def test_without_bias(dev):
    _check(dev, 2, 64, 1028, 3, 3, seed=9, bias=False)


@pytest.mark.parametrize("C,T", [(32, 102400), (64, 51200)])
def test_bench_shapes(dev, C, T):
    _check(dev, 4, C, T, 11, 5, mode="acc", seed=13)


def test_ragged_length_falls_back(dev):
    """T % 4 != 0: the fused kernel declines and the block runs the two launches"""
    from parallelwavegan_b200 import layers, ops

    x, w1, b1, w2, b2 = _inputs(dev, 2, 32, 2049, 3, seed=3)
    with torch.no_grad():
        assert ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=3, dilation=1, slope=SLOPE) is None
        blk = layers.HiFiGANResidualBlock(kernel_size=3, channels=32, dilations=(1, 3, 5)).to(dev)
        y, names = _profiled(lambda: blk(x))
    assert names == ["conv1d_tc"] * 6, names
    ref = x.cpu()
    for i, d in enumerate((1, 3, 5)):
        c1, c2 = blk.convs1[i][1], blk.convs2[i][1]
        xt = torch.nn.functional.conv1d(torch.nn.functional.leaky_relu(ref, SLOPE), c1.weight.cpu(), c1.bias.cpu(), padding=d,
                                        dilation=d)
        ref = torch.nn.functional.conv1d(torch.nn.functional.leaky_relu(xt, SLOPE), c2.weight.cpu(), c2.bias.cpu(), padding=1) + ref
    assert rel_l2(y.cpu(), ref) < 1e-4
    assert max_abs_over_peak(y.cpu(), ref) < 5e-4


@pytest.mark.parametrize("C,T", [(32, 4096), (64, 2048)])
def test_block_uses_fused_pairs(dev, monkeypatch, C, T):
    """HiFiGANResidualBlock at inference: three fused launches, the same result as with the fused op disabled"""
    from parallelwavegan_b200 import layers, ops

    torch.manual_seed(C)
    blk = layers.HiFiGANResidualBlock(kernel_size=7, channels=C, dilations=(1, 3, 5)).to(dev)
    x = torch.randn(4, C, T, device=dev)
    with torch.no_grad():
        out = torch.randn_like(x)
        prev = out.clone()
        y, names = _profiled(lambda: blk(x, out=out, accumulate=True, out_scale=1.0 / 3.0))
        assert names == ["resblock_pair_tc"] * 3, names
        monkeypatch.setattr(ops, "resblock_pair", lambda *a, **k: None)
        y_ref, names_ref = _profiled(lambda: blk(x, out=prev, accumulate=True, out_scale=1.0 / 3.0))
    assert names_ref == ["conv1d_tc"] * 6, names_ref
    assert torch.equal(y, y_ref)


def test_training_keeps_two_launches(dev):
    """under autograd the block runs the differentiable two-conv path"""
    from parallelwavegan_b200 import layers

    blk = layers.HiFiGANResidualBlock(kernel_size=3, channels=32, dilations=(1,)).to(dev)
    x = torch.randn(2, 32, 1024, device=dev, requires_grad=True)
    y, names = _profiled(lambda: blk(x))
    assert "resblock_pair_tc" not in names, names
    y.sum().backward()
    assert x.grad is not None
