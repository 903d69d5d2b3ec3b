"""Streaming the causal Parallel WaveGAN on the GPU (parallelwavegan_b200.streaming.CausalPWGStream): streamed audio is
bit-identical to ``inference`` on the whole utterance for every chunk schedule, the two streaming kernels are
bit-identical to torch reconstructions, slots are independent, graphs replay what eager runs compute, and the
unsupported configurations raise."""
import ctypes as C
import json

import pytest
import torch

from helpers import REL_TOL, golden_weights, load_golden, rel_l2
from oracle import synth
from stream_harness import dev  # noqa: F401

pytestmark = pytest.mark.gpu

# one frame at a time, chunks shorter and longer than the largest layer history (PWG v1: 2048 samples = 8 frames),
# and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [17], "mixed": [1, 7, 2, 33, 5, 1, 12]}
V1 = dict(in_channels=1, out_channels=1, kernel_size=3, layers=30, stacks=3, residual_channels=64, gate_channels=128,
          skip_channels=64, aux_channels=80, aux_context_window=2, use_causal_conv=True, upsample_conditional_features=True,
          upsample_net="ConvInUpsampleNetwork", upsample_params={"upsample_scales": [4, 4, 4, 4]})
CONFIGS = {
    "acw0": dict(aux_context_window=0),
    "acw1": dict(aux_context_window=1),
    "acw2": dict(aux_context_window=2),
    "acw3": dict(aux_context_window=3),
    "upnet": dict(aux_context_window=0, upsample_net="UpsampleNetwork"),
    "k2": dict(kernel_size=2, layers=10, stacks=1, upsample_params={"upsample_scales": [4, 4, 4]}),
}


def _model(dev, config="acw2", weight_norm=True, seed=81, **over):
    from parallelwavegan_b200 import models

    kw = json.loads(json.dumps(dict(V1, **CONFIGS[config], **over)))
    m = models.ParallelWaveGANGenerator(**kw)
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed, 1.0))
    if not weight_norm:
        m.remove_weight_norm()
    return m.to(dev).eval()


def _inputs(m, B, frames, seed):
    c = synth.randn((B, frames, m.aux_channels), seed)
    z = synth.randn((B, 1, frames * m.upsample_factor), seed + 1)
    return c, z


def _stream(st, c, z, schedule, hop):
    outs, j, k = [], 0, 0
    while j < c.shape[1]:
        n = min(schedule[k % len(schedule)], c.shape[1] - j)
        outs.append(st.push(c[:, j:j + n], z[:, :, j * hop:(j + n) * hop]))
        j, k = j + n, k + 1
    return torch.cat(outs, -1)


def _inference(m, c, z):
    """model.inference of each item alone: (B, out_channels, T)"""
    d = next(m.parameters()).device
    with torch.no_grad():
        return torch.stack([m.inference(c=c[b].to(d), x=z[b].t().to(d)).t() for b in range(c.shape[0])])


def _ffma_kernel():
    """the kernel of the last FFMA conv dispatch: 1 conv1d_small_cout_kernel, 2 conv1d_fewcout_long_kernel"""
    from parallelwavegan_b200 import capi

    v = (C.c_int * 6)()
    assert capi.lib().pwgb_debug_get(3, C.cast(v, C.c_void_p), C.sizeof(v)) == 0
    return v[0]


# ------------------------------------------------------------------------------------------------ bit identity
@pytest.mark.parametrize("weight_norm", [True, False])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_stream_bit_identical_to_inference(dev, config, weight_norm):
    from parallelwavegan_b200.streaming import CausalPWGStream

    m = _model(dev, config, weight_norm)
    c, z = _inputs(m, 1, 48, 300)
    ref = _inference(m, c, z)
    assert _ffma_kernel() == 1  # 48 * 256 samples: the 64 -> 1 output conv takes conv1d_small_cout_kernel
    for name, schedule in SCHEDULES.items():
        st = CausalPWGStream(m, batch=1, use_graphs=False)
        y = _stream(st, c.to(dev), z.to(dev), schedule, m.upsample_factor)
        assert _ffma_kernel() == 1
        assert torch.equal(y, ref), (name, rel_l2(y.cpu(), ref.cpu()))


def test_stream_long_utterance(dev):
    """Above B * T = 65536 the whole-utterance output conv switches to conv1d_fewcout_long_kernel, which sums its 64
    inputs in another order; the stream's chunks stay on conv1d_small_cout_kernel.  Everything before that conv is
    still bit-identical, so the difference is that summation order alone."""
    from parallelwavegan_b200.streaming import CausalPWGStream

    m = _model(dev)
    c, z = _inputs(m, 1, 300, 310)
    ref = _inference(m, c, z)
    assert _ffma_kernel() == 2
    st = CausalPWGStream(m, use_graphs=False)
    y = _stream(st, c.to(dev), z.to(dev), [64, 5, 31], m.upsample_factor)
    assert _ffma_kernel() == 1
    assert rel_l2(y.cpu(), ref.cpu()) <= 1e-6


# ------------------------------------------------------------------------------------------------ the two kernels
@pytest.mark.parametrize("t,h_save,h_load", [(256, 2048, 1024), (256, 2, 4), (1024, 512, 0), (512, 0, 2048), (4096, 2048, 2048)])
def test_carry_kernel_bit_for_bit(dev, t, h_save, h_load):
    """pwgb_wnstack_carry against slicing of the packed buffers: rows [t - h, t) (reaching into the halo when t < h)
    saved, and the h rows in front of sample 0 loaded, every other row untouched"""
    from parallelwavegan_b200 import ops

    B, R = 2, 64
    st = ops.WnStack(B, t, R, 128, 64, 80, 3, 1024, dev, causal=True)
    halo = st.desc.halo
    g = torch.Generator(device=dev).manual_seed(t + h_save)
    for x in st.x:  # any bit pattern: the carry is a copy
        x.copy_(torch.randint(-2**31, 2**31 - 1, x.shape, device=dev, dtype=torch.int32, generator=g))
    st.pack_x(torch.randn((B, R, t), device=dev, generator=g))
    st.prev = st.x[0]
    st.cur = 1
    hs = torch.zeros(st.hist_numel(h_save), device=dev, dtype=torch.int32)
    hl = torch.randint(-2**31, 2**31 - 1, (st.hist_numel(h_load),), device=dev, dtype=torch.int32, generator=g)
    before = [x.clone() for x in st.x]
    st.carry(save=(hs, h_save) if h_save else None, load=(hl, h_load) if h_load else None)
    torch.cuda.synchronize()
    planes = [x.view(B * 2 * R // 8, -1, 4) for x in before]  # [plane][row][8 bf16 = 4 int32]
    assert torch.equal(hs.view(B * 2 * R // 8, h_save, 4), planes[0][:, halo + t - h_save: halo + t])
    exp = planes[1].clone()
    exp[:, halo - h_load: halo] = hl.view(B * 2 * R // 8, h_load, 4)
    assert torch.equal(st.x[1].view_as(exp), exp)
    assert torch.equal(st.x[0], before[0])


@pytest.mark.parametrize("n,scale,oc", [(1, 4, None), (2, 4, None), (37, 4, 96), (300, 8, None), (5, 3, None)])
def test_stream_fir_and_carry_bit_for_bit(dev, n, scale, oc):
    """pwgb_upsample_fir_causal_stream_forward against the whole-signal causal stage on [history | x] with its first
    two frames' outputs dropped, and the history the stream's carry hands on against the last two frames"""
    from parallelwavegan_b200 import ops

    B, Cc = 2, 80
    g = torch.Generator(device=dev).manual_seed(n * 10 + scale)
    x = torch.randn((B, Cc, n), device=dev, generator=g)
    hist = torch.randn((B, Cc, 2), device=dev, generator=g)
    fir = torch.randn(2 * scale + 1, device=dev, generator=g)
    y = ops.upsample_fir_causal_stream(x, fir, scale, hist, out_channels=oc)
    xc = torch.cat([hist, x], -1)
    ref = ops.upsample_fir(xc, fir, scale, causal=True)[:, :, 2 * scale:]
    assert torch.equal(y[:, :Cc], ref)
    if oc:
        assert not y[:, Cc:].any()
    ops.stream_carry(ops.stream_carry_table([(x, hist)], dev))
    assert torch.equal(hist, xc[:, :, -2:])


def test_stream_fir_zero_history_equals_the_causal_stage(dev):
    from parallelwavegan_b200 import ops

    g = torch.Generator(device=dev).manual_seed(5)
    x = torch.randn((3, 80, 50), device=dev, generator=g)
    fir = torch.randn(9, device=dev, generator=g)
    y = ops.upsample_fir_causal_stream(x, fir, 4, torch.zeros((240, 2), device=dev))
    assert torch.equal(y, ops.upsample_fir(x, fir, 4, causal=True))


# ------------------------------------------------------------------------------------------------ slots, reset, graphs
def test_batch_slots_are_independent(dev):
    from parallelwavegan_b200.streaming import CausalPWGStream

    m = _model(dev)
    c, z = _inputs(m, 4, 40, 320)
    ref = _inference(m, c, z)
    st = CausalPWGStream(m, batch=4, use_graphs=False)
    y = _stream(st, c.to(dev), z.to(dev), SCHEDULES["mixed"], m.upsample_factor)
    for b in range(4):
        assert torch.equal(y[b], ref[b]), b
    # fp32 conv_in and FIR histories, and (K-1)*d packed hi/lo bf16 rows of R channels per WaveNet layer
    A, R = m.aux_channels, m.conv_layers[0].conv.in_channels
    wn = sum(R * (f.conv.kernel_size[0] - 1) * f.dilation for f in m.conv_layers)
    assert st.state_bytes() == 4 * (A * m.aux_context_window + 2 * A * len(m.upsample_net.upsample.upsample_scales) + wn)


def test_reset_one_slot_mid_stream(dev):
    from parallelwavegan_b200.streaming import CausalPWGStream

    m = _model(dev, "acw3")
    hop = m.upsample_factor
    c, z = _inputs(m, 2, 30, 330)
    c2, z2 = _inputs(m, 2, 20, 340)
    st = CausalPWGStream(m, batch=2, use_graphs=True)
    y1 = _stream(st, c[:, :10].to(dev), z[:, :, :10 * hop].to(dev), [3, 2], hop)
    st.reset(1)  # slot 1 starts a new utterance (c2[1]); slot 0 continues
    cn = torch.stack([c[0, 10:30], c2[1]])
    zn = torch.stack([z[0, :, 10 * hop:], z2[1]])
    y2 = _stream(st, cn.to(dev), zn.to(dev), [1, 6], hop)
    ref0 = _inference(m, c[:1], z[:1])[0]
    ref1 = _inference(m, c2[1:], z2[1:])[0]
    assert torch.equal(torch.cat([y1[0], y2[0]], -1), ref0)
    assert torch.equal(y2[1], ref1)


def test_graph_replay_equals_eager(dev):
    from parallelwavegan_b200.streaming import CausalPWGStream

    m = _model(dev)
    c, z = _inputs(m, 2, 60, 350)
    ys = []
    for graphs in (False, True):
        st = CausalPWGStream(m, batch=2, use_graphs=graphs)
        ys.append(_stream(st, c.to(dev), z.to(dev), SCHEDULES["mixed"], m.upsample_factor))
    assert torch.equal(ys[0], ys[1])
    # noise drawn from the stream's seeded generator: reproducible, graphs or not
    outs = []
    for graphs in (False, True):
        st = CausalPWGStream(m, batch=2, seed=7, use_graphs=graphs)
        outs.append(torch.cat([st.push(c[:, j:j + 4].to(dev)) for j in range(0, 12, 4)], -1))
    assert torch.equal(outs[0], outs[1])


# ------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize("name", ["pwg_causal_v1", "pwg_causal_k2"])
def test_stream_golden(dev, name):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.streaming import CausalPWGStream

    meta, g = load_golden(name)
    m = models.ParallelWaveGANGenerator(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    m = m.to(dev).eval()
    ctx = meta["kwargs"]["aux_context_window"]
    c = synth.randn(meta["c_shape"], meta["c_seed"])[:1, :, ctx: meta["c_shape"][-1] - ctx].transpose(1, 2)
    z = synth.randn(meta["z_shape"], meta["z_seed"])[:1]
    y = _stream(CausalPWGStream(m), c.to(dev), z.to(dev), SCHEDULES["mixed"], m.upsample_factor)
    assert rel_l2(y[0].t().cpu(), g["y_inf"]) < REL_TOL


# ------------------------------------------------------------------------------------------------ refusals
def test_unsupported_configurations_raise(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import CausalPWGStream

    with pytest.raises(PwgbError, match="not causal"):
        CausalPWGStream(_model(dev, use_causal_conv=False))
    for name in ("pwg_causal_small_acw2", "pwg_causal_melgan_up"):  # 8 residual channels / the MelGAN upsampler
        meta, _ = load_golden(name)
        m = models.ParallelWaveGANGenerator(**json.loads(json.dumps(meta["kwargs"]))).to(dev).eval()
        with pytest.raises(PwgbError):
            CausalPWGStream(m)
    with pytest.raises(PwgbError, match="upsample_conditional_features"):
        CausalPWGStream(_model(dev, upsample_conditional_features=False))
    m = _model(dev)
    with pytest.raises(PwgbError, match="train mode"):
        CausalPWGStream(m.train())
    st = CausalPWGStream(m.eval())
    m.train()
    with pytest.raises(PwgbError, match="train mode"):
        st.push(torch.zeros(2, 80))
    m.eval()
