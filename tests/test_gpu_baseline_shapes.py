"""GPU parity at the BASELINE.json shapes (C2 / C3 / C4 / C5) and at tile counts that make every
persistent CTA of the tensor-core kernels loop many times (running ring counters, accumulator-set and
mbarrier-parity wraps).  The GPU computes the full batch; the CPU oracle re-computes a few batch
items (the ops are batch-independent), so the whole file costs seconds of host time.
Tolerance: rel-L2 <= 1e-3 and max-abs <= 1e-3 of peak (north_star), far tighter where noted."""
import pytest
import torch
import torch.nn.functional as F

from helpers import REL_TOL, max_abs_over_peak, rel_l2
from oracle import ref_ops, synth
from oracle.ref_ops import fold_spectral_norm_eval, fold_weight_norm

pytestmark = pytest.mark.gpu

TC_TOL = 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def _synth_load(m, seed, gain):
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed, gain)
    m.load_state_dict(sd)
    return sd


def _check(y, ref, tag, tol=REL_TOL):
    e, p = rel_l2(y, ref), max_abs_over_peak(y, ref)
    print(f"{tag}: rel-L2 {e:.2e} max-abs/peak {p:.2e}")
    assert e < tol and p < 5 * tol, (tag, e, p)


def test_c2_hifigan_v1_16x80x400(dev):
    """BASELINE configs[1] (the bench workload): 16x80x400 -> 16x1x102400; 43 tiles per CTA."""
    import bench
    from parallelwavegan_b200 import models

    m = models.HiFiGANGenerator(**bench.CFG)
    sd = _synth_load(m, 1234, 1.15)
    m.remove_weight_norm()
    m = m.eval().to(dev)
    c = synth.randn((16, 80, 400), 100)
    with torch.no_grad():
        y = m(c.to(dev)).cpu()
    assert tuple(y.shape) == (16, 1, 102400)
    w = fold_weight_norm(sd)
    for i in (0, 15):
        ref = ref_ops.hifigan_generator(w, c[i : i + 1], dict(bench.CFG, negative_slope=0.1))
        _check(y[i : i + 1], ref, f"C2 utterance {i}")


def test_c4_mb_melgan_32x80x400_pqmf(dev):
    """BASELINE configs[3]: multi-band MelGAN v2 + PQMF synthesis, 32x80x400 -> 32x1x120000."""
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.layers import PQMF

    cfg = dict(ref_ops.MB_MELGAN_V2)
    kw = dict(in_channels=80, out_channels=4, kernel_size=7, channels=384, upsample_scales=[5, 5, 3], stack_kernel_size=3, stacks=4)
    m = models.MelGANGenerator(**kw)
    sd = _synth_load(m, 77, 1.1)
    m = m.eval().to(dev)
    pq = PQMF(4).to(dev)
    c = synth.randn((32, 80, 400), 101)
    with torch.no_grad():
        sub = m(c.to(dev))
        y = pq.synthesis(sub).cpu()
    assert tuple(y.shape) == (32, 1, 120000)
    w = fold_weight_norm(sd)
    an, sy = ref_ops.pqmf_filters(4)
    for i in (0, 31):
        rs = ref_ops.melgan_generator(w, c[i : i + 1], cfg)
        _check(sub[i : i + 1].cpu(), rs, f"C4 sub-bands {i}")
        _check(y[i : i + 1], ref_ops.pqmf_synthesis(rs, sy), f"C4 PQMF {i}")


@pytest.mark.parametrize("batch", [16, 64])
def test_c3_pwg_generator_forward(dev, batch):
    """PWG v1 generator at B x 25600 (B = 64 is the C3 per-GPU batch): 30 fused layers, every
    dilation 1..512, 100..400 tiles per CTA."""
    from parallelwavegan_b200 import models

    m = models.ParallelWaveGANGenerator()
    sd = _synth_load(m, 31, 1.0)
    m = m.eval().to(dev)
    T = 25600
    z = synth.randn((batch, 1, T), 102)
    c = synth.randn((batch, 80, T // 256 + 4), 103)
    with torch.no_grad():
        y = m(z.to(dev), c.to(dev)).cpu()
    w = fold_weight_norm(sd)
    cfg = dict(ref_ops.PWG_V1)
    for i in (0, batch - 1):
        ref = ref_ops.pwg_generator(w, z[i : i + 1], c[i : i + 1], cfg)
        _check(y[i : i + 1], ref, f"PWG B={batch} item {i}")


def test_c5_msmpd_16x8192_full_tensors(dev):
    """HiFi-GAN MSD + MPD at the C5 batch: EVERY feature map compared in full with the oracle
    (not a fingerprint) for two batch items."""
    from parallelwavegan_b200 import models

    m = models.HiFiGANMultiScaleMultiPeriodDiscriminator()
    sd = _synth_load(m, 4321, 1.4)
    m = m.eval().to(dev)
    x = synth.randn((16, 1, 8192), 104, 0.3)
    with torch.no_grad():
        outs = m(x.to(dev))
    w = fold_weight_norm(fold_spectral_norm_eval(sd))
    items = [0, 15]
    ref = ref_ops.hifigan_msmpd(w, x[items])
    assert len(outs) == len(ref) == 8
    n = 0
    for di, (o, r) in enumerate(zip(outs, ref)):
        assert len(o) == len(r)
        for li, (a, b) in enumerate(zip(o, r)):
            a = a[items].cpu()
            assert tuple(a.shape) == tuple(b.shape), (di, li)
            _check(a, b, f"C5 D{di} layer {li} {tuple(b.shape)}")
            n += 1
    assert n == 3 * 8 + 5 * 6


@pytest.mark.parametrize(
    "cin,cout,k,dil,T,B,res",
    [
        (64, 64, 3, 1, 51200, 16, True),     # 3200 work items of 256 rows: > 21 per CTA, both accumulator sets wrap
        (32, 32, 3, 3, 102400, 16, True),    # 6400 items
        (128, 128, 11, 5, 25600, 16, False),  # tensor-bound shape of the bench
        (256, 256, 3, 1, 3200, 16, True),    # MT = 1, single accumulator set
    ],
)
def test_conv1d_tc_many_tiles(dev, cin, cout, k, dil, T, B, res):
    from parallelwavegan_b200 import ops

    pad = (k - 1) // 2 * dil
    x = synth.randn((B, cin, T), 1)
    w = synth.randn((cout, cin, k), 2, 1.0 / (cin * k) ** 0.5)
    b = synth.randn((cout,), 3, 0.1)
    r = synth.randn((B, cout, T), 4) if res else None
    ops.PROFILE = []
    try:
        y = ops.conv1d(x.to(dev), w.to(dev), b.to(dev), padding=pad, dilation=dil, pre_slope=0.1,
                       residual=r.to(dev) if res else None)
        torch.cuda.synchronize()
        assert ops.PROFILE[0][0] == "conv1d_tc"
    finally:
        ops.PROFILE = None
    y = y.cpu()
    for i in (0, B // 2, B - 1):
        ref = F.conv1d(F.leaky_relu(x[i : i + 1], 0.1), w, b, padding=pad, dilation=dil)
        if res:
            ref = ref + r[i : i + 1]
        _check(y[i : i + 1], ref, f"conv1d_tc {cin}->{cout} k{k} item {i}", TC_TOL)


def test_conv_transpose_column_chunks_c2(dev):
    """HiFi-GAN v1 first upsampler at the C2 size: 512 -> 256, k16 s8 is a poly-phase conv with
    256 * 8 = 2048 accumulator columns, i.e. 8 column chunks sharing one launch."""
    from parallelwavegan_b200 import ops

    x = synth.randn((16, 512, 400), 5)
    w = synth.randn((512, 256, 16), 6, 0.02)
    b = synth.randn((256,), 7, 0.1)
    y = ops.conv_transpose1d(x.to(dev), w.to(dev), b.to(dev), stride=8, padding=4, pre_slope=0.1).cpu()
    for i in (0, 15):
        ref = F.conv_transpose1d(F.leaky_relu(x[i : i + 1], 0.1), w, b, stride=8, padding=4)
        _check(y[i : i + 1], ref, f"conv_transpose item {i}", TC_TOL)


@pytest.mark.parametrize(
    "cin,cout,k,dil,T,B",
    [
        (128, 128, 11, 5, 2048, 16),   # HiFi-GAN G stage-2 resblock conv at the C5 crop (8192 / 4)
        (512, 512, 3, 1, 256, 16),     # wide, short: split-K over (batch, chunk) items
        (1024, 1024, 5, 2, 104, 16),   # MPD p=2 last layer as a dilated flat conv (hifigan.py:354-381)
    ],
)
def test_wgrad_tc_c5_sizes(dev, cin, cout, k, dil, T, B):
    from parallelwavegan_b200 import ops

    pad = (k - 1) // 2 * dil
    x = synth.randn((B, cin, T), 8)
    gy = synth.randn((B, cout, T), 9)
    ops.PROFILE = []
    try:
        dw = ops.conv1d_wgrad(x.to(dev), gy.to(dev), (cout, cin, k), padding=pad, dilation=dil)
        torch.cuda.synchronize()
        assert ops.PROFILE[0][0] == "conv1d_wgrad_tc"
    finally:
        ops.PROFILE = None
    w = torch.zeros(cout, cin, k, requires_grad=True)
    with torch.enable_grad():
        F.conv1d(x, w, None, padding=pad, dilation=dil).backward(gy)
    _check(dw.cpu(), w.grad, f"wgrad_tc {cin}->{cout} k{k}", TC_TOL)


@pytest.mark.parametrize(
    "cin,cout,k,groups,T,B,expect",
    [
        (1024, 1024, 41, 16, 128, 16, "conv1d_wgrad_tc"),  # MSD layer 5 (grouped, stride 1) at the C5 batch
        (256, 128, 21, 4, 4096, 4, "conv1d_wgrad_tc"),     # MSD layer 1 after space-to-depth (cin_g 64, cout_g 32)
        (1, 128, 15, 1, 8192, 16, "conv1d_wgrad"),         # MSD input conv: narrow kernel, 131k-long reduction
        (1024, 1, 3, 1, 128, 16, "conv1d_wgrad"),          # logit conv: narrow kernel
    ],
)
def test_wgrad_grouped_and_narrow_c5_sizes(dev, cin, cout, k, groups, T, B, expect):
    from parallelwavegan_b200 import ops

    pad = (k - 1) // 2
    x = synth.randn((B, cin, T), 18)
    gy = synth.randn((B, cout, T), 19)
    ops.PROFILE = []
    try:
        dw = ops.conv1d_wgrad(x.to(dev), gy.to(dev), (cout, cin // groups, k), padding=pad, groups=groups)
        torch.cuda.synchronize()
        assert ops.PROFILE[0][0] == expect
    finally:
        ops.PROFILE = None
    w = torch.zeros(cout, cin // groups, k, requires_grad=True)
    with torch.enable_grad():
        F.conv1d(x, w, None, padding=pad, groups=groups).backward(gy)
    _check(dw.cpu(), w.grad, f"wgrad {cin}->{cout} k{k} g{groups}", TC_TOL)


def test_wide_short_convs_single_launch(dev):
    """1024-channel discriminator layers on ~100-sample rows: every (group, 128-column chunk, batch, tile) item runs in
    ONE launch (dense 1024 -> 1024 k5 as the MPD does it on the flat period view, and the grouped MSD k41 layer)."""
    from parallelwavegan_b200 import capi, ops

    for cin, cout, k, groups, dil, T, B in ((1024, 1024, 5, 1, 2, 104, 16), (1024, 1024, 41, 16, 1, 128, 16), (512, 1024, 3, 1, 1, 52, 3)):
        pad = (k - 1) // 2 * dil
        x = synth.randn((B, cin, T), 28)
        w = synth.randn((cout, cin // groups, k), 29, 1.0 / (cin // groups * k) ** 0.5)
        b = synth.randn((cout,), 30, 0.1)
        capi.reset_launch_count()
        ops.PROFILE = []
        try:
            y = ops.conv1d(x.to(dev), w.to(dev), b.to(dev), padding=pad, dilation=dil, groups=groups, post_act="lrelu", post_slope=0.1)
            torch.cuda.synchronize()
            assert ops.PROFILE[0][0] == "conv1d_tc"
        finally:
            ops.PROFILE = None
        assert capi.launch_count() == 2  # weight pack + ONE conv launch
        ref = F.leaky_relu(F.conv1d(x, w, b, padding=pad, dilation=dil, groups=groups), 0.1)
        _check(y.cpu(), ref, f"wide conv {cin}->{cout} k{k} g{groups}", TC_TOL)
