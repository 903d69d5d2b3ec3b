"""The 128- and 256-channel ResBlock conv pairs (pwgb_resblock_pair_packed_forward): conv1's epilogue writes the
intermediate as conv2's packed bf16 hi/lo operand image and conv2 lands it with tensor copies.  The operands, the MMA
order and the epilogues are those of the two fp32 conv1d_tc launches it replaces, so every output must be
bit-identical to them.  pwgb_debug_set(1, 8) turns the packed pair off (the two-launch path); ops.PROFILE shows which
path ran."""
import pytest
import torch

pytestmark = pytest.mark.gpu

SLOPE = 0.1


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _profiled(fn):
    from parallelwavegan_b200 import ops

    ops.PROFILE = []
    try:
        y = fn()
        torch.cuda.synchronize()
        return y, [p[0] for p in ops.PROFILE]
    finally:
        ops.PROFILE = None


class _Unpacked:
    """the two-launch path for the duration of the block"""

    def __enter__(self):
        from parallelwavegan_b200 import capi

        capi.lib().pwgb_debug_set(1, 8)

    def __exit__(self, *exc):
        from parallelwavegan_b200 import capi

        capi.lib().pwgb_debug_set(1, 0)


def _inputs(dev, B, C, T, k, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, C, T, device=dev, generator=g)
    w1 = torch.randn(C, C, k, device=dev, generator=g) / (C * k) ** 0.5
    w2 = torch.randn(C, C, k, device=dev, generator=g) / (C * k) ** 0.5
    b1 = 0.1 * torch.randn(C, device=dev, generator=g)
    b2 = 0.1 * torch.randn(C, device=dev, generator=g)
    return x, w1, b1, w2, b2


def _two_launches(x, w1, b1, w2, b2, k, d, **tail):
    from parallelwavegan_b200 import ops

    xt = ops.conv1d(x, w1, b1, dilation=d, padding=(k - 1) // 2 * d, pre_slope=SLOPE)
    return ops.conv1d(xt, w2, b2, padding=(k - 1) // 2, pre_slope=SLOPE, residual=x, **tail)


def _check(dev, B, C, T, k, d, mode, seed):
    from parallelwavegan_b200 import ops

    x, w1, b1, w2, b2 = _inputs(dev, B, C, T, k, seed)
    prev = torch.randn(B, C, T, device=dev, generator=torch.Generator(device=dev).manual_seed(seed + 1))
    kw = {} if mode == "plain" else dict(out_scale=1.0 / 3.0, accumulate=mode == "acc")
    with torch.no_grad():
        out_p = prev.clone() if mode != "plain" else None
        y_p, names = _profiled(lambda: ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=k, dilation=d, slope=SLOPE, out=out_p, **kw))
        out_r = prev.clone() if mode != "plain" else None
        y_r, names_r = _profiled(lambda: _two_launches(x, w1, b1, w2, b2, k, d, out=out_r, **kw))
    assert names == ["resblock_pair_packed_tc"], names
    assert names_r == ["conv1d_tc", "conv1d_tc"], names_r
    if out_p is not None:
        assert y_p is out_p
    assert torch.equal(y_p, y_r)


@pytest.mark.parametrize("C", [128, 256])
@pytest.mark.parametrize("k", [3, 7, 11])
@pytest.mark.parametrize("d", [1, 3, 5])
@pytest.mark.parametrize("T", [1024, 1060, 52])
@pytest.mark.parametrize("mode", ["plain", "out", "acc"])
def test_pair_bit_identical(dev, C, k, d, T, mode):
    # T: whole 128-row tiles, a ragged last tile (a multiple of 4), one tile shorter than 128 rows
    B = 1 if (k + d + T) % 2 else 3
    _check(dev, B, C, T, k, d, mode, seed=C + 10 * k + d + T)


@pytest.mark.parametrize("C,T", [(256, 3200), (128, 25600)])
def test_bench_shapes(dev, C, T):
    """the headline's shapes: many tiles per CTA, the rings and the residual phases wrap many times"""
    _check(dev, 16, C, T, 11, 5, "acc", seed=7)


def test_plan_frees_raw_stages(dev):
    """conv2 lands its operand images from the packed intermediate: no raw stages, their bytes are weight stages"""
    import ctypes as C

    from parallelwavegan_b200 import capi, ops

    x, w1, b1, w2, b2 = _inputs(dev, 2, 128, 1024, 11, seed=3)
    v = (C.c_int * 8)()
    with torch.no_grad():
        ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=11, dilation=5, slope=SLOPE)
        torch.cuda.synchronize()
        assert capi.lib().pwgb_debug_get(1, C.cast(v, C.c_void_p), C.sizeof(v)) == 0
        packed = list(v)
        with _Unpacked():
            _two_launches(x, w1, b1, w2, b2, 11, 5)
            torch.cuda.synchronize()
            assert capi.lib().pwgb_debug_get(1, C.cast(v, C.c_void_p), C.sizeof(v)) == 0
        unpacked = list(v)
    # {MT, na, nb, ns, staged, tma_act, win_mode, nco}
    assert unpacked[3] > 0 and unpacked[4] == 1, unpacked
    assert packed[3] == 0 and packed[4] == 1 and packed[2] > unpacked[2], (packed, unpacked)


def test_ragged_length_keeps_two_launches(dev):
    """T % 4 != 0: conv2 cannot stage its residual, the pair declines and the block runs the two fp32 launches"""
    from parallelwavegan_b200 import layers, ops

    x, w1, b1, w2, b2 = _inputs(dev, 2, 128, 1026, 3, seed=4)
    with torch.no_grad():
        assert ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=3, dilation=1, slope=SLOPE) is None
        blk = layers.HiFiGANResidualBlock(kernel_size=3, channels=128, dilations=(1, 3)).to(dev)
        _, names = _profiled(lambda: blk(x))
    assert names == ["conv1d_tc"] * 4, names


def test_switch_turns_the_pair_off(dev):
    from parallelwavegan_b200 import ops

    x, w1, b1, w2, b2 = _inputs(dev, 1, 256, 512, 3, seed=5)
    with torch.no_grad(), _Unpacked():
        assert ops.resblock_pair(x, w1, b1, w2, b2, kernel_size=3, dilation=1, slope=SLOPE) is None


def _both_paths(fn):
    with torch.no_grad():
        y, names = _profiled(fn)
        with _Unpacked():
            y_ref, names_ref = _profiled(fn)
    assert "resblock_pair_packed_tc" in names and "resblock_pair_packed_tc" not in names_ref
    assert torch.equal(y, y_ref)
    return names, names_ref


def test_hifigan_v1_generator(dev):
    from parallelwavegan_b200 import models

    torch.manual_seed(0)
    m = models.HiFiGANGenerator().to(dev).eval()
    mel = torch.randn(2, 80, 48, device=dev)
    names, names_ref = _both_paths(lambda: m(mel))
    # each packed record stands for the two conv1d_tc launches of its pair
    assert names.count("resblock_pair_packed_tc") == 18, names
    assert names_ref.count("conv1d_tc") == names.count("conv1d_tc") + 36


def test_uhifigan_generator(dev):
    from parallelwavegan_b200 import models

    # the opencpop recipe: 32 .. 512 channels, 300 samples per frame; its 128- and 256-channel MRF levels, on both sides
    # of the U, take the packed pairs
    torch.manual_seed(1)
    m = models.UHiFiGANGenerator(channels=32, downsample_scales=(5, 5, 4, 3), downsample_kernel_sizes=(10, 10, 8, 6),
                                 upsample_scales=(3, 4, 5, 5), upsample_kernel_sizes=(6, 8, 10, 10)).to(dev).eval()
    mel = torch.randn(2, 80, 40, device=dev)
    exc = torch.randn(2, 1, 40 * 300, device=dev)
    names, _ = _both_paths(lambda: m(mel, None, exc))
    assert names.count("resblock_pair_packed_tc") == 36, names


def test_graphed_generator_replay(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.decode import GraphedGenerator

    torch.manual_seed(2)
    m = models.HiFiGANGenerator().to(dev).eval()
    m.remove_weight_norm()
    g = GraphedGenerator(m)
    for seed in (3, 4):  # the second call replays the captured graph on new mels
        mel = torch.randn(2, 80, 32, device=dev, generator=torch.Generator(device=dev).manual_seed(seed))
        with torch.no_grad():
            y = g(mel).clone()
            with _Unpacked():
                y_ref = m(mel)
        assert torch.equal(y, y_ref)
