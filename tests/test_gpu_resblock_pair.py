"""The fused ResBlock conv pair (rb_pair_split_kernel, csrc/resblock_tc.cu) against the two tensor-core conv launches it
replaces.  The fused kernel uses the same weight images, bf16x3 split and MMA order into every accumulator, and the same
epilogue order, so the outputs must be bit-identical; on grid data it must also reproduce the exact bf16x3 reference
(oracle/bf16x3.py).  ops.PROFILE shows which path ran."""
import pytest
import torch

from helpers import max_abs_over_peak, rel_l2
from oracle import bf16x3 as E

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


@pytest.mark.parametrize("C,k,d,B,T", [(64, 3, 1, 16, 16384), (64, 11, 5, 3, 51200), (32, 7, 3, 16, 16384), (32, 11, 5, 2, 102400)])
def test_many_tiles_per_cta(dev, C, k, d, B, T):
    """several passes of the persistent grid (hundreds to thousands of tiles, not a multiple of the grid): the H_FULL /
    H_FREE, ring and residual phases wrap many times"""
    _check(dev, B, C, T, k, d, mode="acc", seed=T + B)


@pytest.mark.parametrize("C,k,d", [(32, 11, 5), (64, 11, 5), (32, 3, 1), (64, 3, 1)])
@pytest.mark.parametrize("T", [4, 8, 12, 48])
def test_shorter_than_halo(dev, C, k, d, T):
    _check(dev, 3, C, T, k, d, seed=T)


@pytest.mark.parametrize("C,k,d", [(32, 7, 5), (64, 11, 3), (32, 11, 3), (64, 7, 5)])
@pytest.mark.parametrize("mode", ["out", "acc"])
def test_last_pair_writes_out(dev, C, k, d, mode):
    _check(dev, 2, C, 4100, k, d, mode=mode, seed=5)


def test_without_bias(dev):
    for C, k, d in [(64, 3, 3), (32, 7, 3), (64, 7, 3)]:
        _check(dev, 2, C, 1028, k, d, seed=9 + C + k, bias=False)


@pytest.mark.parametrize("C", [32, 64])
def test_empty_batch(dev, C):
    from parallelwavegan_b200 import ops

    x, w1, b1, w2, b2 = _inputs(dev, 0, C, 1024, 3, seed=1)
    with torch.no_grad():
        y, names = _profiled(lambda: ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=3, dilation=1, slope=SLOPE))
    assert y is not None and y.shape == x.shape and names == [], names


@pytest.mark.parametrize("C,k,d,mode", [(32, 11, 5, "acc"), (64, 11, 5, "acc"), (64, 3, 1, "plain"), (32, 7, 3, "out")])
def test_exact_on_grid_data(dev, C, k, d, mode):
    """grid data (every bf16x3 product and partial sum exact in fp32): the fused kernel equals the exact reference"""
    B, T = 2, 4100
    g = torch.Generator().manual_seed(C * 1000 + k * 10 + d)
    for hmax, z in [(1, 0.0), (1, 0.4), (1, 0.6), (1, 0.75), (1, 0.85), (1, 0.92)]:
        x = E.grid_values((B, C, T), g, 1.0, hmax, z)
        w1 = E.grid_values((C, C, k), g, 2.0 ** -3, hmax, z)
        b1 = E.grid_values((C,), g, 2.0 ** -3, 3)
        w2 = E.grid_values((C, C, k), g, 2.0 ** -1, hmax, z, lo=False)
        b2 = E.grid_values((C,), g, 2.0 ** -1, 3)
        prev = E.grid_values((B, C, T), g, 2.0, 3) if mode == "acc" else None
        ref, ex = E.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=0.5, out_scale=0.5, prev=prev)
        if ex.ok:
            break
    assert ex.ok, "no grid data passes the exactness guard"
    from parallelwavegan_b200 import ops

    out = None
    if mode == "acc":
        out = prev.to(dev)
    elif mode == "out":
        out = torch.full((B, C, T), float("nan"), device=dev)
    with torch.no_grad():
        y, names = _profiled(lambda: ops.resblock_pair(x.to(dev), w1.to(dev), b1.to(dev), w2.to(dev), b2.to(dev), kernel_size=k,
                                                       dilation=d, slope=0.5, out=out, accumulate=mode == "acc", out_scale=0.5))
    assert names == ["resblock_pair_tc"], names
    assert torch.equal(y.cpu(), ref)


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


def _block_against_unfused(monkeypatch, dev, C, T, k, dilations, seed, acc):
    """HiFiGANResidualBlock at inference (with acc: out += x' / 3), bit-identical to the same block with the fused op
    disabled (two conv1d_tc launches per pair); returns the launches of the first run"""
    from parallelwavegan_b200 import layers, ops

    torch.manual_seed(seed)
    blk = layers.HiFiGANResidualBlock(kernel_size=k, channels=C, dilations=dilations).to(dev)
    x = torch.randn(4, C, T, device=dev)
    kw = dict(accumulate=True, out_scale=1.0 / 3.0) if acc else {}
    with torch.no_grad():
        out = torch.randn_like(x) if acc else None
        prev = out.clone() if acc else None
        y, names = _profiled(lambda: blk(x, out=out, **kw))
        monkeypatch.setattr(ops, "resblock_pair", lambda *a, **k: None)
        y_ref, names_ref = _profiled(lambda: blk(x, out=prev, **kw))
    assert names_ref == ["conv1d_tc"] * (2 * len(dilations)), names_ref
    assert torch.equal(y, y_ref)
    return names


@pytest.mark.parametrize("C,T", [(32, 4096), (64, 2048)])
def test_block_uses_fused_pairs(dev, monkeypatch, C, T):
    """the last block of an MRF sum: three fused launches"""
    names = _block_against_unfused(monkeypatch, dev, C, T, 7, (1, 3, 5), seed=C, acc=True)
    assert names == ["resblock_pair_tc"] * 3, names


@pytest.mark.parametrize("C,T", [(32, 4096), (64, 2048)])
def test_block_one_launch_per_pair(dev, monkeypatch, C, T):
    names = _block_against_unfused(monkeypatch, dev, C, T, 11, (1, 3, 5), seed=C + 1, acc=False)
    assert names == ["resblock_pair_tc"] * 3, names


def test_block_wide_halo_pair_keeps_two_launches(dev, monkeypatch):
    """at 64 channels and k = 11, conv1's halo at d = 6 is too wide for the fused kernel's plan: that pair runs the two
    launches and the d = 1 pair stays fused"""
    names = _block_against_unfused(monkeypatch, dev, 64, 2048, 11, (1, 6), seed=6, acc=False)
    assert names == ["resblock_pair_tc", "conv1d_tc", "conv1d_tc"], names


def test_training_keeps_two_launches(dev):
    """under autograd the block runs the differentiable two-conv path"""
    from parallelwavegan_b200 import layers

    blk = layers.HiFiGANResidualBlock(kernel_size=3, channels=32, dilations=(1,)).to(dev)
    x = torch.randn(2, 32, 1024, device=dev, requires_grad=True)
    y, names = _profiled(lambda: blk(x))
    assert "resblock_pair_tc" not in names, names
    y.sum().backward()
    assert x.grad is not None
