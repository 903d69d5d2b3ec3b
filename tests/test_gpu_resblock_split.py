"""The conv-split fused ResBlock pair (rb_pair_split_kernel, csrc/resblock_tc.cu) against the lockstep kernel
(pwgb_debug_set(3, 1)) and against the two tensor-core conv launches it replaces.  All three use the same weight images,
bf16x3 split, MMA order into every accumulator and epilogue order, so the outputs must be bit-identical; on grid data
the split kernel must also reproduce the exact bf16x3 reference (oracle/bf16x3.py)."""
import pytest
import torch

from oracle import bf16x3 as E

pytestmark = pytest.mark.gpu

SLOPE = 0.1
V1 = [(C, k, d) for C in (32, 64) for k in (3, 7, 11) for d in (1, 3, 5)]


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


def _fused(x, w1, b1, w2, b2, k, d, lockstep, out=None, **kw):
    from parallelwavegan_b200 import capi, ops

    capi.lib().pwgb_debug_set(3, int(lockstep))
    try:
        B, C, T = x.shape
        plan = ops.resblock_pair_plan(C, T, k, d, batch=B)
        assert plan is not None and plan["variant"] == ("lockstep" if lockstep else "split"), plan
        y, names = _profiled(lambda: ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=SLOPE, out=out, **kw))
    finally:
        capi.lib().pwgb_debug_set(3, 0)
    assert names == ["resblock_pair_tc"], names  # one launch per pair
    return y


def _two_launches(x, w1, b1, w2, b2, k, d, out=None, accumulate=False, out_scale=1.0):
    from parallelwavegan_b200 import ops

    xt = ops.conv1d(x, w1, b1, dilation=d, padding=(k - 1) // 2 * d, pre_slope=SLOPE)
    return ops.conv1d(xt, w2, b2, padding=(k - 1) // 2, pre_slope=SLOPE, residual=x, out=out, accumulate=accumulate,
                      out_scale=out_scale)


def _check(dev, B, C, T, k, d, mode="plain", seed=0, bias=True, two_launches=True):
    x, w1, b1, w2, b2 = _inputs(dev, B, C, T, k, seed, bias)
    kw = {}
    prev = None
    if mode != "plain":  # last pair of a block: out (+)= x' / 3
        prev = torch.randn(B, C, T, device=dev, generator=torch.Generator(device=dev).manual_seed(seed + 1))
        kw = dict(out_scale=1.0 / 3.0, accumulate=mode == "acc")
    with torch.no_grad():
        outs = [prev.clone() if prev is not None else None for _ in range(3)]
        y_s = _fused(x, w1, b1, w2, b2, k, d, False, out=outs[0], **kw)
        y_l = _fused(x, w1, b1, w2, b2, k, d, True, out=outs[1], **kw)
        if two_launches:
            y_r, names = _profiled(lambda: _two_launches(x, w1, b1, w2, b2, k, d, out=outs[2], **kw))
            assert names == ["conv1d_tc", "conv1d_tc"], names
    if prev is not None:
        assert y_s is outs[0]
    assert torch.equal(y_s, y_l)
    if two_launches:
        assert torch.equal(y_s, y_r)


@pytest.mark.parametrize("C,k,d", V1)
def test_v1_pairs_bit_identical(dev, C, k, d):
    # T = 2052: not a multiple of any tile's output rows (124 / 120 / 116 at 64 channels, 252 / 248 / 244 at 32)
    _check(dev, 2, C, 2052, k, d, seed=100 + C + k + d)


@pytest.mark.parametrize("C,k,d,B,T", [(64, 3, 1, 16, 16384), (64, 11, 5, 3, 51200), (32, 7, 3, 16, 16384), (32, 11, 5, 2, 102400)])
def test_many_tiles_per_cta(dev, C, k, d, B, T):
    """several passes of the persistent grid (hundreds to thousands of tiles, not a multiple of the grid): the H_FULL /
    H_FREE, ring and residual phases wrap many times"""
    _check(dev, B, C, T, k, d, mode="acc", seed=T + B)


@pytest.mark.parametrize("C,k,d", [(32, 11, 5), (64, 11, 5), (64, 3, 1)])
@pytest.mark.parametrize("T", [4, 12, 48])
def test_shorter_than_halo(dev, C, k, d, T):
    _check(dev, 3, C, T, k, d, seed=T)


@pytest.mark.parametrize("C,k,d", [(32, 11, 3), (64, 7, 5)])
@pytest.mark.parametrize("mode", ["out", "acc"])
def test_last_pair_writes_out(dev, C, k, d, mode):
    _check(dev, 2, C, 4100, k, d, mode=mode, seed=7)


@pytest.mark.parametrize("C", [32, 64])
def test_without_bias(dev, C):
    _check(dev, 2, C, 1028, 7, 3, seed=11, bias=False)


@pytest.mark.parametrize("C", [32, 64])
def test_empty_batch(dev, C):
    from parallelwavegan_b200 import ops

    x, w1, b1, w2, b2 = _inputs(dev, 0, C, 1024, 3, seed=1)
    with torch.no_grad():
        y, names = _profiled(lambda: ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=3, dilation=1, slope=SLOPE))
    assert y is not None and y.shape == x.shape and names == [], names


@pytest.mark.parametrize("C,k,d,mode", [(32, 11, 5, "acc"), (64, 11, 5, "acc"), (64, 3, 1, "plain"), (32, 7, 3, "out")])
def test_exact_on_grid_data(dev, C, k, d, mode):
    """grid data (every bf16x3 product and partial sum exact in fp32): the split kernel equals the exact reference"""
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
        plan = ops.resblock_pair_plan(C, T, k, d, batch=B)
        assert plan["variant"] == "split", plan
        y, names = _profiled(lambda: ops.resblock_pair(x.to(dev), w1.to(dev), b1.to(dev), w2.to(dev), b2.to(dev), kernel_size=k,
                                                       dilation=d, slope=0.5, out=out, accumulate=mode == "acc", out_scale=0.5))
    assert names == ["resblock_pair_tc"], names
    assert torch.equal(y.cpu(), ref)


@pytest.mark.parametrize("C,T", [(32, 4096), (64, 2048)])
def test_block_one_launch_per_pair(dev, C, T):
    """HiFiGANResidualBlock at inference: one split launch per pair, bit-identical to the forced lockstep kernel"""
    from parallelwavegan_b200 import capi, layers

    torch.manual_seed(C + 1)
    blk = layers.HiFiGANResidualBlock(kernel_size=11, channels=C, dilations=(1, 3, 5)).to(dev)
    x = torch.randn(4, C, T, device=dev)
    with torch.no_grad():
        y, names = _profiled(lambda: blk(x))
        capi.lib().pwgb_debug_set(3, 1)
        try:
            y_l, names_l = _profiled(lambda: blk(x))
        finally:
            capi.lib().pwgb_debug_set(3, 0)
    assert names == ["resblock_pair_tc"] * 3 and names_l == names, (names, names_l)
    assert torch.equal(y, y_l)
