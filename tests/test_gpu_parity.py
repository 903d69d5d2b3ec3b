"""GPU parity tests: CUDA path (through the C ABI) vs golden vectors from the real reference
and vs the CPU oracle on the same seeded inputs.  Tolerance: rel-L2 <= 1e-3 (north_star);
the fp32 FFMA kernels are expected to sit near 1e-6."""
import json

import pytest
import torch
import torch.nn.functional as F

from helpers import REL_TOL, golden_effective_weights, golden_weights, load_golden, max_abs_over_peak, rel_l2
from oracle import ref_ops, synth

pytestmark = pytest.mark.gpu

FP32_TOL = 2e-5  # exact-arithmetic (FFMA) kernels: summation-order noise only


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import __graft_entry__

    __graft_entry__.build()
    return torch.device("cuda:0")


def test_conv_golden_cases(dev):
    from parallelwavegan_b200 import ops

    meta, g = load_golden("conv_cases")
    for case in meta["cases"]:
        i = case["idx"]
        x = synth.randn((2, case["cin"], case["T"]), 200 + i).to(dev)
        b = synth.randn((case["cout"],), 400 + i, 0.1).to(dev)
        if case["op"] == "conv1d":
            w = synth.randn((case["cout"], case["cin"] // case["groups"], case["k"]), 300 + i, 0.3).to(dev)
            y = ops.conv1d(x, w, b, stride=case["stride"], padding=case["padding"], dilation=case["dilation"], groups=case["groups"])
        else:
            s = case["stride"]
            w = synth.randn((case["cin"], case["cout"], case["k"]), 300 + i, 0.3).to(dev)
            y = ops.conv_transpose1d(x, w, b, stride=s, padding=s // 2 + s % 2, output_padding=s % 2)
        assert tuple(y.shape) == tuple(g[f"y{i}"].shape), case
        assert rel_l2(y.cpu(), g[f"y{i}"]) < FP32_TOL, case


@pytest.mark.parametrize(
    "cin,cout,k,stride,dil,groups,pad,mode,T,B",
    [
        (64, 64, 3, 1, 1, 1, (1, 1), "zero", 1000, 3),
        (32, 32, 11, 1, 5, 1, (25, 25), "zero", 777, 2),
        (48, 48, 3, 1, 9, 1, (9, 9), "reflect", 300, 2),
        (16, 24, 5, 1, 2, 1, (8, 0), "replicate", 129, 2),
        (128, 128, 41, 4, 1, 4, (20, 20), "zero", 2048, 2),
        (128, 256, 41, 4, 1, 16, (20, 20), "zero", 513, 2),
        (1, 128, 15, 1, 1, 1, (7, 7), "zero", 4096, 2),
        (64, 1, 7, 1, 1, 1, (3, 3), "zero", 5000, 2),
        (20, 4, 7, 1, 1, 1, (3, 3), "reflect", 260, 2),
        (80, 80, 5, 1, 1, 1, (0, 0), "zero", 104, 2),
        (3, 5, 1, 1, 1, 1, (0, 0), "zero", 1, 1),
    ],
)
def test_conv1d_fused_options(dev, cin, cout, k, stride, dil, groups, pad, mode, T, B):
    from parallelwavegan_b200 import ops

    x = synth.randn((B, cin, T), 1)
    w = synth.randn((cout, cin // groups, k), 2, 1.0 / (cin // groups * k) ** 0.5)
    b = synth.randn((cout,), 3, 0.1)
    xa = F.leaky_relu(x, 0.1)
    if mode == "zero":
        xp = F.pad(xa, pad)
    else:
        xp = F.pad(xa, pad, mode=mode)
    conv = F.conv1d(xp, w, b, stride=stride, dilation=dil, groups=groups)
    res = synth.randn(conv.shape, 4)
    prev = synth.randn(conv.shape, 5)
    ref = prev + 0.5 * (torch.tanh(conv) + res)
    out = prev.clone().to(dev)
    y = ops.conv1d(x.to(dev), w.to(dev), b.to(dev), stride=stride, padding=pad, dilation=dil, groups=groups,
                   pad_mode=mode, pre_slope=0.1, post_act="tanh", residual=res.to(dev), out_scale=0.5, out=out, accumulate=True)
    assert y.data_ptr() == out.data_ptr()
    assert rel_l2(y.cpu(), ref) < FP32_TOL
    # plain form
    y2 = ops.conv1d(x.to(dev), w.to(dev), None, stride=stride, padding=pad, dilation=dil, groups=groups, pad_mode=mode)
    xp2 = F.pad(x, pad) if mode == "zero" else F.pad(x, pad, mode=mode)
    assert rel_l2(y2.cpu(), F.conv1d(xp2, w, None, stride=stride, dilation=dil, groups=groups)) < FP32_TOL


@pytest.mark.parametrize("period", [2, 3, 5, 7, 11])
def test_conv1d_period_view(dev, period):
    """MPD layer semantics (hifigan.py:354-381): reflect-extend to a multiple of P, view (B,C,T/P,P),
    Conv2d (5,1) stride (3,1) pad (2,0); then a second layer on the 4-D result."""
    from parallelwavegan_b200 import ops

    B, T = 2, 1000 + period - 3
    x = synth.randn((B, 1, T), 11)
    w1 = synth.randn((32, 1, 5, 1), 12, 0.4)
    b1 = synth.randn((32,), 13, 0.1)
    w2 = synth.randn((64, 32, 5, 1), 14, 0.08)
    xr = x
    if T % period:
        xr = F.pad(x, (0, period - T % period), "reflect")
    xv = xr.view(B, 1, -1, period)
    r1 = F.leaky_relu(F.conv2d(xv, w1, b1, stride=(3, 1), padding=(2, 0)), 0.1)
    r2 = F.conv2d(r1, w2, None, stride=(3, 1), padding=(2, 0))
    y1 = ops.conv1d(x.to(dev), w1.to(dev), b1.to(dev), stride=3, padding=2, period=period, post_act="lrelu", post_slope=0.1)
    assert tuple(y1.shape) == tuple(r1.shape)
    assert rel_l2(y1.cpu(), r1) < FP32_TOL
    y2 = ops.conv1d(y1, w2.to(dev), None, stride=3, padding=2, period=period)
    assert rel_l2(y2.cpu(), r2) < FP32_TOL


def _load_mirror(name, dev):
    from parallelwavegan_b200 import models

    meta, g = load_golden(name)
    cls = {"hifigan_generator": models.HiFiGANGenerator, "melgan_generator": models.MelGANGenerator,
           "pwg_generator": getattr(models, "ParallelWaveGANGenerator", None)}[meta["kind"]]
    if cls is None:
        pytest.skip("not built yet")
    m = cls(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    return meta, g, m.eval().to(dev)


@pytest.mark.parametrize("name", ["hifigan_small", "hifigan_v1", "hifigan_odd", "hifigan_causal"])
@pytest.mark.parametrize("weight_norm", [True, False])
def test_hifigan_generator_vs_reference(dev, name, weight_norm):
    meta, g, m = _load_mirror(name, dev)
    if not weight_norm:
        m.remove_weight_norm()
    c = synth.randn(meta["c_shape"], meta["c_seed"]).to(dev)
    with torch.no_grad():
        y = m(c)
        y_inf = m.inference(c[0].t())
    assert tuple(y.shape) == tuple(g["y"].shape)
    assert rel_l2(y.cpu(), g["y"]) < REL_TOL and max_abs_over_peak(y.cpu(), g["y"]) < REL_TOL
    assert rel_l2(y_inf.cpu(), g["y_inf"]) < REL_TOL
    # and against the travelling oracle, same weights
    kw = meta["kwargs"]
    ref = ref_ops.hifigan_generator(golden_effective_weights(meta), c.cpu(), dict(kw, negative_slope=kw["nonlinear_activation_params"]["negative_slope"]))
    assert rel_l2(y.cpu(), ref) < REL_TOL


@pytest.mark.parametrize("name", ["mb_melgan_v2", "melgan_small", "melgan_causal"])
def test_melgan_generator_vs_reference(dev, name):
    from parallelwavegan_b200.layers import PQMF

    meta, g, m = _load_mirror(name, dev)
    c = synth.randn(meta["c_shape"], meta["c_seed"]).to(dev)
    with torch.no_grad():
        y = m(c)
    assert rel_l2(y.cpu(), g["y"]) < REL_TOL and max_abs_over_peak(y.cpu(), g["y"]) < REL_TOL
    if meta.get("pqmf_subbands"):
        pq = PQMF(meta["pqmf_subbands"]).to(dev)
        with torch.no_grad():
            yp = pq.synthesis(y)
            m.pqmf = pq
            y_inf = m.inference(c[0].t())
        assert rel_l2(yp.cpu(), g["y_pqmf"]) < REL_TOL
        assert rel_l2(y_inf.cpu(), g["y_inf"]) < REL_TOL


@pytest.mark.parametrize("name", ["hifigan_causal", "melgan_causal"])
def test_causal_generators_are_causal(dev, name):
    """test/test_hifigan.py:198-226, test/test_melgan.py (causal): perturbing the second half of the
    conditioning leaves the first half of the waveform bit-identical."""
    meta, g, m = _load_mirror(name, dev)
    B, C, T = 2, meta["c_shape"][1], 32
    c = synth.randn((B, C, T), 77).to(dev)
    c2 = c.clone()
    c2[..., T // 2:] = synth.randn((B, C, T - T // 2), 78).to(dev)
    with torch.no_grad():
        y, y2 = m(c), m(c2)
    hop = y.shape[-1] // T
    assert y.shape[-1] == T * hop
    assert torch.equal(y[..., : T // 2 * hop], y2[..., : T // 2 * hop])
    assert not torch.equal(y[..., T // 2 * hop:], y2[..., T // 2 * hop:])


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_pqmf_vs_reference(dev, n):
    from parallelwavegan_b200.layers import PQMF

    meta, g = load_golden(f"pqmf_{n}")
    pq = PQMF(n).to(dev)
    assert torch.equal(pq.analysis_filter.cpu(), g["analysis_filter"])
    assert torch.equal(pq.synthesis_filter.cpu(), g["synthesis_filter"])
    x = synth.randn(meta["x_shape"], meta["x_seed"]).to(dev)
    a = pq.analysis(x)
    assert tuple(a.shape) == tuple(g["analysis"].shape)
    assert rel_l2(a.cpu(), g["analysis"]) < FP32_TOL
    s = pq.synthesis(g["analysis"].to(dev))
    assert tuple(s.shape) == tuple(g["synthesis"].shape)
    assert rel_l2(s.cpu(), g["synthesis"]) < FP32_TOL


@pytest.mark.parametrize("n", [2, 4, 8])
def test_pqmf_band_interleave_bit_exact(dev, n):
    """north_star: "bit-exact for PQMF integer banding".  With small-integer signals and
    filters every partial sum is exact in fp32, so the poly-phase kernels must reproduce the
    reference's zero-stuff / stride-N index arithmetic (pqmf.py:130-131, 146-149) bit for bit."""
    from parallelwavegan_b200.layers import PQMF

    pq = PQMF(n).to(dev)
    gen = torch.Generator().manual_seed(n)
    an = torch.randint(-3, 4, (n, 1, 63), generator=gen).float()
    sy = torch.randint(-3, 4, (1, n, 63), generator=gen).float()
    pq.analysis_filter.copy_(an)
    pq.synthesis_filter.copy_(sy)
    x = torch.randint(-8, 9, (3, 1, 40 * n + 0), generator=gen).float()
    a_ref = ref_ops.pqmf_analysis(x, an)
    a = pq.analysis(x.to(dev))
    assert torch.equal(a.cpu(), a_ref)
    sub = torch.randint(-8, 9, (3, n, 50), generator=gen).float()
    s_ref = ref_ops.pqmf_synthesis(sub, sy)
    s = pq.synthesis(sub.to(dev))
    assert torch.equal(s.cpu(), s_ref)


TC_TOL = 1e-4  # bf16x3 split: ~2^-16 per product, fp32 accumulation


@pytest.mark.parametrize(
    "cin,cout,k,dil,T,B,mode",
    [
        (32, 32, 3, 1, 300, 2, "zero"),
        (32, 16, 1, 1, 128, 1, "zero"),
        (64, 64, 7, 3, 1000, 2, "zero"),
        (128, 128, 11, 5, 700, 2, "zero"),
        (256, 256, 3, 1, 513, 1, "zero"),
        (256, 256, 11, 5, 400, 2, "zero"),
        (64, 128, 3, 2, 129, 3, "zero"),
        (96, 192, 3, 9, 260, 2, "reflect"),
        (192, 192, 3, 27, 300, 1, "reflect"),
        (64, 64, 3, 4, 5, 2, "replicate"),
        (32, 48, 5, 1, 2049, 1, "zero"),
    ],
)
def test_conv1d_tcgen05_path(dev, cin, cout, k, dil, T, B, mode):
    """tensor-core bf16x3 path vs the oracle (ATen fp32 on CPU) and vs the FFMA kernel."""
    import ctypes as C

    from parallelwavegan_b200 import capi, ops

    pad = (k - 1) // 2 * dil
    x = synth.randn((B, cin, T), 1)
    w = synth.randn((cout, cin, k), 2, 1.0 / (cin * k) ** 0.5)
    b = synth.randn((cout,), 3, 0.1)
    xa = F.leaky_relu(x, 0.1)
    xp = F.pad(xa, (pad, pad)) if mode == "zero" else F.pad(xa, (pad, pad), mode=mode)
    conv = F.conv1d(xp, w, b, dilation=dil)
    res = synth.randn(conv.shape, 4)
    prev = synth.randn(conv.shape, 5)
    ref = prev + 0.5 * (conv + res)
    kw = dict(padding=pad, dilation=dil, pad_mode=mode, pre_slope=0.1, residual=res.to(dev), out_scale=0.5, accumulate=True)
    d = capi.Conv1dDesc(batch=B, cin=cin, cout=cout, t_in=T, t_out=T, kernel=k, stride=1, dilation=dil, groups=1,
                        pad_left=pad, pad_mode=ops._PAD[mode], period=1, t_valid=T, pre_slope=0.1, out_scale=0.5)
    assert capi.lib().pwgb_conv1d_tc_supported(C.byref(d)) == 1
    old = ops.ENGINE
    try:
        ops.ENGINE = "auto"
        ops.PROFILE = []
        y_tc = ops.conv1d(x.to(dev), w.to(dev), b.to(dev), out=prev.clone().to(dev), **kw)
        torch.cuda.synchronize()
        assert ops.PROFILE[0][0] == "conv1d_tc"
        ops.PROFILE = None
        ops.ENGINE = "simt"
        y_ff = ops.conv1d(x.to(dev), w.to(dev), b.to(dev), out=prev.clone().to(dev), **kw)
    finally:
        ops.ENGINE = old
        ops.PROFILE = None
    e_tc, e_ff = rel_l2(y_tc.cpu(), ref), rel_l2(y_ff.cpu(), ref)
    print(f"tc rel {e_tc:.2e} simt rel {e_ff:.2e} maxabs/peak {max_abs_over_peak(y_tc.cpu(), ref):.2e}")
    assert e_ff < FP32_TOL
    assert e_tc < TC_TOL, (e_tc, e_ff)
    assert max_abs_over_peak(y_tc.cpu(), ref) < TC_TOL * 5


@pytest.mark.parametrize("name", ["pwg_v1", "pwg_small"])
def test_pwg_generator_vs_reference(dev, name):
    meta, g, m = _load_mirror(name, dev)
    kw = meta["kwargs"]
    c = synth.randn(meta["c_shape"], meta["c_seed"]).to(dev)
    z = synth.randn(meta["z_shape"], meta["z_seed"]).to(dev)
    ctx = kw["aux_context_window"]
    with torch.no_grad():
        c_up = m.upsample_net(c)
        y = m(z, c)
        y_inf = m.inference(c=c[0, :, ctx : c.shape[-1] - ctx].t(), x=z[0].t())
        x0 = m.first_conv.weight  # noqa: F841  (container only)
    assert rel_l2(c_up[:, :, :512].cpu(), g["c_up"]) < FP32_TOL * 5
    assert tuple(y.shape) == tuple(g["y"].shape)
    assert rel_l2(y.cpu(), g["y"]) < REL_TOL and max_abs_over_peak(y.cpu(), g["y"]) < REL_TOL
    assert rel_l2(y_inf.cpu(), g["y_inf"]) < REL_TOL
    cfg = dict(kw, upsample_scales=kw["upsample_params"]["upsample_scales"])
    ref = ref_ops.pwg_generator(golden_effective_weights(meta), z.cpu(), c.cpu(), cfg)
    assert rel_l2(y.cpu(), ref) < REL_TOL


@pytest.mark.parametrize("dilation,T,B", [(1, 700, 2), (16, 1000, 2), (64, 515, 1), (128, 1500, 2), (512, 2100, 1)])
@pytest.mark.parametrize("engine", ["auto", "simt"])
def test_wavenet_layer(dev, dilation, T, B, engine):
    """One WaveNetResidualBlock (PWG v1 sizes) vs the oracle, both engines; dilation 128/512
    exercise the per-tap window mode of the tensor-core kernel."""
    from parallelwavegan_b200 import layers, ops

    blk = layers.WaveNetResidualBlock(dilation=dilation)
    spec = [(k, tuple(v.shape)) for k, v in blk.state_dict().items()]
    sd = synth.synth_state_dict(spec, 40 + dilation, 1.0)
    blk.load_state_dict(sd)
    blk = blk.to(dev)
    x = synth.randn((B, 64, T), 1)
    c = synth.randn((B, 80, T), 2)
    sk0 = synth.randn((B, 64, T), 3)
    w = {f"b.{k}": v for k, v in sd.items()}
    xr, sr = ref_ops.wavenet_residual_block(w, "b", x, c, dilation, 3)
    cp = torch.zeros(B, 96, T)
    cp[:, :80] = c
    skips = sk0.clone().to(dev)
    old = ops.ENGINE
    try:
        ops.ENGINE = engine
        ops.PROFILE = []
        with torch.no_grad():
            xo, so = blk(x.to(dev), cp.to(dev), skips)
        torch.cuda.synchronize()
        names = [p[0] for p in ops.PROFILE]
    finally:
        ops.ENGINE = old
        ops.PROFILE = None
    if engine == "auto":
        assert names == ["wavenet_layer_tc"]
    tol = TC_TOL if engine == "auto" else FP32_TOL
    assert rel_l2(xo.cpu(), xr) < tol
    assert rel_l2(so.cpu(), sk0 + sr) < tol


@pytest.mark.parametrize("dilation,T,B", [(1, 700, 2), (16, 1000, 2), (64, 515, 1), (128, 1500, 2), (512, 2100, 1), (2, 128 * 150, 3)])
@pytest.mark.parametrize("skips_init,write_x", [(False, True), (True, True), (False, False)])
def test_wavenet_fused_layer_packed(dev, dilation, T, B, skips_init, write_x):
    """The ONE-kernel fused layer on the packed (bf16 hi/lo operand layout) residual stream vs the oracle:
    pack -> pwgb_wnstack_layer_forward -> unpack.  Covers ragged tails (T % 128 != 0), every tap window
    reaching into the zero halo, skip initialisation and the last-layer form (no residual output);
    the last case gives every CTA several tiles (both ring phases wrap)."""
    from parallelwavegan_b200 import layers, ops

    blk = layers.WaveNetResidualBlock(dilation=dilation)
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in blk.state_dict().items()], 40 + dilation, 1.0)
    blk.load_state_dict(sd)
    blk = blk.to(dev)
    x = synth.randn((B, 64, T), 1)
    c = synth.randn((B, 80, T), 2)
    sk0 = synth.randn((B, 64, T), 3)
    w = {f"b.{k}": v for k, v in sd.items()}
    xr, sr = ref_ops.wavenet_residual_block(w, "b", x, c, dilation, 3)
    assert ops.WnStack.supported(B, T, 64, 128, 64, 80, 3, 512)
    st = ops.WnStack(B, T, 64, 128, 64, 80, 3, 512, dev)
    st.pack_c(c.to(dev))
    st.pack_x(x.to(dev))
    assert rel_l2(st.unpack_x().cpu(), x) < 1e-5  # the packed stream carries 16+ mantissa bits
    skips = sk0.clone().to(dev)
    with torch.no_grad():
        packed, bso = ops.wavenet_packed_weights(layers.effective_weight(blk.conv), layers.effective_weight(blk.conv1x1_aux),
                                                 layers.effective_weight(blk.conv1x1_skip), layers.effective_weight(blk.conv1x1_out),
                                                 blk.conv1x1_skip.bias, blk.conv1x1_out.bias, 80)
        st.layer(packed, blk.conv.bias, bso, dilation, skips, skips_init=skips_init, write_x=write_x)
        torch.cuda.synchronize()
        xo = st.unpack_x().cpu()
    if write_x:
        assert rel_l2(xo, xr) < TC_TOL and max_abs_over_peak(xo, xr) < 5 * TC_TOL
    else:
        assert rel_l2(xo, x) < 1e-5  # stream untouched
    assert rel_l2(skips.cpu(), sr if skips_init else sk0 + sr) < TC_TOL
    # the zero halo of the written buffer must still be zero (the next layer's padding)
    raw = st.x[st.cur].view(torch.int32)
    planes = raw.view(B * 2 * 8, -1, 4)
    assert int(planes[:, :512].abs().sum()) == 0 and int(planes[:, 512 + T:].abs().sum()) == 0


@pytest.mark.parametrize("R,G,S,A", [(32, 64, 32, 80), (96, 128, 32, 64), (32, 128, 96, 80)])
def test_wavenet_fused_layer_packed_other_channel_counts(dev, R, G, S, A):
    """The fused layer for channel counts other than the PWG v1 ones (run-time channel loops of the kernel:
    residual / skip halves wider than one 64-column register block, a conditioning width that is a multiple of 32)."""
    from parallelwavegan_b200 import layers, ops

    B, T, dilation = 2, 900, 4
    blk = layers.WaveNetResidualBlock(residual_channels=R, gate_channels=G, skip_channels=S, aux_channels=A, dilation=dilation)
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in blk.state_dict().items()], 90 + R, 1.0)
    blk.load_state_dict(sd)
    blk = blk.to(dev)
    x, c, sk0 = synth.randn((B, R, T), 1), synth.randn((B, A, T), 2), synth.randn((B, S, T), 3)
    xr, sr = ref_ops.wavenet_residual_block({f"b.{k}": v for k, v in sd.items()}, "b", x, c, dilation, 3)
    assert ops.WnStack.supported(B, T, R, G, S, A, 3, 16)
    st = ops.WnStack(B, T, R, G, S, A, 3, 16, dev)
    st.pack_c(c.to(dev))
    st.pack_x(x.to(dev))
    skips = sk0.clone().to(dev)
    with torch.no_grad():
        packed, bso = ops.wavenet_packed_weights(layers.effective_weight(blk.conv), layers.effective_weight(blk.conv1x1_aux),
                                                 layers.effective_weight(blk.conv1x1_skip), layers.effective_weight(blk.conv1x1_out),
                                                 blk.conv1x1_skip.bias, blk.conv1x1_out.bias, A)
        st.layer(packed, blk.conv.bias, bso, dilation, skips)
        torch.cuda.synchronize()
        xo = st.unpack_x().cpu()
    assert rel_l2(xo, xr) < TC_TOL and rel_l2(skips.cpu(), sk0 + sr) < TC_TOL


@pytest.mark.parametrize("update", ["inplace_op", "fused_optimizer", "load_state_dict"])
def test_pwg_forward_sees_weight_updates(dev, update):
    """Packed operand images are cached per layer, keyed on the LEAF parameters (weight_g / weight_v / bias):
    a second no-grad forward after an in-place update, a fused-optimizer step or load_state_dict must use the
    new weights (round-1 advisor finding: the cache was keyed on weight-norm temporaries)."""
    from parallelwavegan_b200 import models, optimizers

    kw = dict(layers=6, stacks=3)
    m = models.ParallelWaveGANGenerator(**kw)
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 5, 1.0)
    m.load_state_dict(sd)
    m = m.to(dev)
    z = synth.randn((2, 1, 2560), 6)
    c = synth.randn((2, 80, 14), 7)
    cfg = dict(ref_ops.PWG_V1, **kw)

    def check():
        with torch.no_grad():
            y = m(z.to(dev), c.to(dev)).cpu()
        cur = {k: v.detach().cpu() for k, v in m.state_dict().items()}
        ref = ref_ops.pwg_generator(ref_ops.fold_weight_norm(cur), z, c, cfg)
        assert rel_l2(y, ref) < REL_TOL

    check()
    if update == "inplace_op":
        with torch.no_grad():
            for n, p in m.named_parameters():
                if n.endswith("weight_g"):
                    p.mul_(1.3)
                elif n.endswith("bias"):
                    p.add_(0.05)
    elif update == "fused_optimizer":
        opt = optimizers.RAdam(m.parameters(), lr=5e-2)
        for i, p in enumerate(m.parameters()):
            p.grad = synth.randn(tuple(p.shape), 100 + i).to(dev)
        for _ in range(6):
            opt.step()
    else:
        sd2 = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 55, 1.1)
        m.load_state_dict(sd2)
    check()


def test_upsample_fir(dev):
    from parallelwavegan_b200 import ops

    x = synth.randn((3, 7, 33), 5)
    for s in (2, 4, 5):
        f = synth.randn((2 * s + 1,), 6 + s, 0.3)
        ref = torch.repeat_interleave(x, s, dim=-1)
        ref = F.conv1d(ref.reshape(21, 1, -1), f.reshape(1, 1, -1), padding=s).reshape(3, 7, -1)
        y = ops.upsample_fir(x.to(dev), f.to(dev), s)
        assert rel_l2(y.cpu(), ref) < FP32_TOL
        yp = ops.upsample_fir(x.to(dev), f.to(dev), s, out_channels=32)
        assert tuple(yp.shape) == (3, 32, 33 * s)
        assert rel_l2(yp[:, :7].cpu(), ref) < FP32_TOL and float(yp[:, 7:].abs().max()) == 0.0


def test_graphed_decode_matches_eager(dev):
    """CUDA-graph replay of the generator (decode driver) == eager forward, bit for bit; utterance sharding."""
    from parallelwavegan_b200 import decode

    meta, g, m = _load_mirror("hifigan_small", dev)
    m.remove_weight_norm()
    mels = [synth.randn((n, 80), 900 + n) for n in (12, 20, 12, 31, 20)]
    ours = decode.decode_utterances(m, mels, rank=0, world=1, use_graphs=True)
    for i, mel in enumerate(mels):
        with torch.no_grad():
            ref = m.inference(mel.to(dev))
        assert torch.equal(ours[i], ref), i
    part = decode.decode_utterances(m, mels, rank=1, world=2, use_graphs=False)
    assert sorted(part) == [1, 3]


def test_decoder_pcm16_normalize_and_buckets(dev):
    """Decode driver (bin/decode.py:214-243 on the GPU): on-device normalize_before + transpose, equal-length
    batching bit-identical to ``inference``, PCM16 by libsndfile's rule, async D2H; bucketed mode is exact away from
    the utterance end."""
    import numpy as np

    from parallelwavegan_b200 import decode

    meta, g, m = _load_mirror("hifigan_small", dev)
    m.remove_weight_norm()
    m.register_buffer("mean", synth.randn((80,), 70, 0.3).to(dev))
    m.register_buffer("scale", (synth.randn((80,), 71, 0.1).abs() + 0.5).to(dev))
    mels = [synth.randn((n, 80), 900 + k).numpy() for k, n in enumerate((40, 52, 40, 63, 52, 40))]
    dec = decode.Decoder(m, use_graphs=True, max_batch=2)
    wav = dec.decode(mels, normalize_before=True, to_pcm16=True)
    flt = dec.decode(mels, normalize_before=True, to_pcm16=False)
    for i, mel in enumerate(mels):
        with torch.no_grad():
            ref = m.inference(torch.from_numpy(mel).to(dev), normalize_before=True)
        assert torch.equal(flt[i], ref), i
        exp = np.clip(np.rint(ref[:, 0].cpu().numpy() * np.float32(32767.0)), -32768, 32767).astype(np.int16)
        assert wav[i].dtype == np.int16 and wav[i].shape == exp.shape and np.array_equal(wav[i], exp), i
    # length buckets (approximate at the tail only): compare everything further than one receptive field from the end
    decb = decode.Decoder(m, use_graphs=False, max_batch=8, exact=False, bucket_frames=16)
    fb = decb.decode(mels, normalize_before=True, to_pcm16=False)
    hop = 256
    for i, mel in enumerate(mels):
        n = mel.shape[0] * hop
        assert fb[i].shape == flt[i].shape
        keep = n - 30 * hop  # the generator's receptive field is ~25 frames on each side
        assert rel_l2(fb[i][:keep].cpu(), flt[i][:keep].cpu()) < 1e-5, i


def test_decoder_parallel_wavegan_path(dev):
    """Decoder dispatch for ParallelWaveGANGenerator: replicate-padded conditioning + noise as static graph inputs;
    with the noise pinned the result equals ``inference(c, x)``."""
    from parallelwavegan_b200 import decode

    meta, g, m = _load_mirror("pwg_small", dev)
    hop = m.upsample_factor
    mels = [synth.randn((n, m.aux_channels), 950 + k) for k, n in enumerate((9, 14, 9))]
    noises = {i: synth.randn((mel.shape[0] * hop, 1), 980 + i) for i, mel in enumerate(mels)}
    dec = decode.Decoder(m, use_graphs=True, max_batch=4, seed=3)
    out = dec.decode(mels, to_pcm16=False, noises=noises)
    for i, mel in enumerate(mels):
        with torch.no_grad():
            ref = m.inference(c=mel.to(dev), x=noises[i].to(dev))
        assert tuple(out[i].shape) == tuple(ref.shape)
        assert rel_l2(out[i].cpu(), ref.cpu()) < 1e-6, i
