"""Streaming the centred Parallel WaveGAN with a fixed lookahead on the GPU (parallelwavegan_b200.streaming.
PWGLookaheadStream): for every slot cat(pushes, flush) is bit-identical to [zeros(delay) | inference] for every chunk
schedule, the lookahead WaveNet layer and the masked FIR stage chunked over [history | chunk] are bit-identical to the
centred whole-signal kernels, slots are independent across reset and flush, graphs replay what eager runs compute, and
the unsupported configurations raise."""
import ctypes as C
import json

import pytest
import torch

from helpers import REL_TOL, golden_weights, load_golden, rel_l2
from oracle import synth
from stream_harness import dev  # noqa: F401

pytestmark = pytest.mark.gpu

SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
V1 = dict(in_channels=1, out_channels=1, kernel_size=3, layers=30, stacks=3, residual_channels=64, gate_channels=128,
          skip_channels=64, aux_channels=80, aux_context_window=2, use_causal_conv=False, upsample_conditional_features=True,
          upsample_net="ConvInUpsampleNetwork", upsample_params={"upsample_scales": [4, 4, 4, 4]})


def _model(dev, weight_norm=True, seed=91, **over):
    from parallelwavegan_b200 import models

    m = models.ParallelWaveGANGenerator(**json.loads(json.dumps(dict(V1, **over))))
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed, 1.0))
    if not weight_norm:
        m.remove_weight_norm()
    return m.to(dev).eval()


def _golden_model(dev, name="pwg_v1"):
    from parallelwavegan_b200 import models

    meta, g = load_golden(name)
    m = models.ParallelWaveGANGenerator(**meta["kwargs"])
    m.load_state_dict(golden_weights(meta), strict=True)
    ctx = meta["kwargs"]["aux_context_window"]
    c = synth.randn(meta["c_shape"], meta["c_seed"])
    c = c[:, :, ctx:c.shape[-1] - ctx].transpose(1, 2).contiguous()  # (1, frames, aux)
    z = synth.randn(meta["z_shape"], meta["z_seed"])
    return m.to(dev).eval(), c, z, g


def _inputs(m, B, frames, seed):
    return synth.randn((B, frames, m.aux_channels), seed), synth.randn((B, 1, frames * m.upsample_factor), seed + 1)


def _stream(st, c, z, schedule, hop, flush=True):
    outs, j, k = [], 0, 0
    while j < c.shape[1]:
        n = min(schedule[k % len(schedule)], c.shape[1] - j)
        outs.append(st.push(c[:, j:j + n], z[:, :, j * hop:(j + n) * hop]))
        j, k = j + n, k + 1
    if flush:
        outs.append(st.flush())
    return torch.cat(outs, -1)


def _expected(m, c, z, delay):
    """[zeros(delay) | model.inference] of each item alone: (B, out_channels, delay + T)"""
    d = next(m.parameters()).device
    with torch.no_grad():
        y = torch.stack([m.inference(c=c[b].to(d), x=z[b].t().to(d)).t() for b in range(c.shape[0])])
    return torch.cat([y.new_zeros(y.shape[:-1] + (delay,)), y], -1)


def _ffma_kernel():
    """the kernel of the last FFMA conv dispatch: 1 conv1d_small_cout_kernel, 2 conv1d_fewcout_long_kernel"""
    from parallelwavegan_b200 import capi

    v = (C.c_int * 6)()
    assert capi.lib().pwgb_debug_get(3, C.cast(v, C.c_void_p), C.sizeof(v)) == 0
    return v[0]


# ------------------------------------------------------------------------------------------------ bit identity
@pytest.mark.parametrize("which", ["golden", "v1_wn", "v1_plain"])
def test_stream_bit_identical_to_inference(dev, which):
    from parallelwavegan_b200.streaming import PWGLookaheadStream

    if which == "golden":
        m, c, z, _ = _golden_model(dev)
        c, z = c.repeat(1, 4, 1), z.repeat(1, 1, 4)  # 40 frames
    else:
        m = _model(dev, weight_norm=which == "v1_wn")
        c, z = _inputs(m, 1, 40, 400)
    st = PWGLookaheadStream(m, use_graphs=False)
    assert st.delay == 3920
    ref = _expected(m, c, z, st.delay)
    assert _ffma_kernel() == 1  # 40 * 256 samples: the 64 -> 1 output conv takes conv1d_small_cout_kernel
    for name, schedule in SCHEDULES.items():
        y = _stream(st, c.to(dev), z.to(dev), schedule, m.upsample_factor)
        assert _ffma_kernel() == 1
        assert torch.equal(y, ref), (which, name, rel_l2(y.cpu(), ref.cpu()))


@pytest.mark.parametrize("frames", [1, 2])
def test_utterances_shorter_than_the_delay(dev, frames):
    from parallelwavegan_b200.streaming import PWGLookaheadStream

    m = _model(dev)
    c, z = _inputs(m, 1, frames, 410 + frames)
    st = PWGLookaheadStream(m, use_graphs=False)
    ref = _expected(m, c, z, st.delay)
    for schedule in (SCHEDULES["ones"], SCHEDULES["long"]):
        assert torch.equal(_stream(st, c.to(dev), z.to(dev), schedule, m.upsample_factor), ref)


def test_golden_reference_output(dev):
    """the stored output of the real reference's inference"""
    from parallelwavegan_b200.streaming import PWGLookaheadStream

    m, c, z, g = _golden_model(dev)
    st = PWGLookaheadStream(m)
    y = _stream(st, c.to(dev), z.to(dev), SCHEDULES["mixed"], m.upsample_factor)[0, :, st.delay:]
    assert rel_l2(y.t().cpu(), g["y_inf"]) < REL_TOL


def test_stream_long_utterance(dev):
    """Above B * T = 65536 the whole-utterance output conv sums its 64 inputs in another order (§3.2)"""
    from parallelwavegan_b200.streaming import PWGLookaheadStream

    m = _model(dev)
    c, z = _inputs(m, 1, 300, 420)
    st = PWGLookaheadStream(m)
    ref = _expected(m, c, z, st.delay)
    assert _ffma_kernel() == 2
    y = _stream(st, c.to(dev), z.to(dev), [64, 5, 31], m.upsample_factor)
    assert rel_l2(y.cpu(), ref.cpu()) <= 1e-6


# ------------------------------------------------------------------------------------------------ the kernels
def _wn_weights(dev, R, G, S, A, K, seed):
    from parallelwavegan_b200 import ops

    g = torch.Generator(device=dev).manual_seed(seed)
    r = lambda *s: torch.randn(s, device=dev, generator=g) * 0.3  # noqa: E731
    packed, bso = ops.wavenet_packed_weights(r(G, R, K), r(G, A, 1), r(S, G // 2, 1), r(R, G // 2, 1), r(S), r(R), A)
    return packed, r(G), bso


@pytest.mark.parametrize("dilation", [1, 8, 64])
def test_lookahead_layer_bit_for_bit(dev, dilation):
    """pwgb_wnstack_layer_stream_ext_forward chunked over [history | chunk] with the mask equals the centred
    pwgb_wnstack_layer_forward on the whole signal, for x' and the skips; slot 1 runs 37 samples behind slot 0 (mixed
    frame counters), and the flush pushes zero rows with the end set"""
    from parallelwavegan_b200 import ops

    B, R, G, S, A, K, Tw = 2, 64, 128, 64, 80, 3, 1000
    lag = [0, 37]
    rd = (K - 1) // 2 * dilation
    packed, b_conv, bso = _wn_weights(dev, R, G, S, A, K, dilation)
    g = torch.Generator(device=dev).manual_seed(7 + dilation)
    x = torch.randn((B, R, Tw), device=dev, generator=g)
    c = torch.randn((B, A, Tw), device=dev, generator=g)
    whole = ops.WnStack(B, Tw, R, G, S, A, K, 64, dev)
    whole.pack_x(x)
    whole.pack_c(c)
    skw = torch.empty((B, S, Tw), device=dev)
    whole.layer(packed, b_conv, bso, dilation, skw, skips_init=True)
    xw = whole.unpack_x()

    frame = torch.tensor([-l for l in lag], device=dev, dtype=torch.int32)
    end = torch.full((B,), Tw, device=dev, dtype=torch.int32)
    hist = torch.zeros(B * R * (K - 1) * dilation, device=dev, dtype=torch.int32)
    chist = torch.zeros((B, A, rd), device=dev)
    stacks, xo, so = {}, [], []
    total = Tw + rd + max(lag)
    g0, k = 0, 0
    sched = [100, 37, 256, 5, 300]
    while g0 < total:
        T = min(sched[k % len(sched)], total - g0)
        st = stacks.get(T) or stacks.setdefault(T, ops.WnStack(B, T, R, G, S, A, K, 64, dev, lookahead=True))
        xi = torch.zeros((B, R, T), device=dev)
        ci = torch.zeros((B, A, T), device=dev)
        for b in range(B):
            lo, hi = max(g0 - lag[b], 0), min(g0 + T - lag[b], Tw)
            if hi > lo:
                xi[b, :, lo + lag[b] - g0:hi + lag[b] - g0] = x[b, :, lo:hi]
                ci[b, :, lo + lag[b] - g0:hi + lag[b] - g0] = c[b, :, lo:hi]
        st.cur, st.prev = 0, None
        st.pack_x(xi)
        cw = torch.cat([chist, ci], -1)
        chist = cw[:, :, T:].contiguous()
        cpk, rows = st.pack_c_window(cw)
        H = (K - 1) * dilation
        st.carry(load=(hist, H))
        sk = torch.empty((B, S, T), device=dev)
        st.layer_stream(packed, b_conv, bso, dilation, cpk, rows, 0, sk, 0, (frame, end, 1, rd), skips_init=True)
        st.carry(save=(hist, H))
        xo.append(st.unpack_x())
        so.append(sk)
        frame += T
        g0, k = g0 + T, k + 1
    xo, so = torch.cat(xo, -1), torch.cat(so, -1)
    for b in range(B):
        o = lag[b] + rd
        assert torch.equal(xo[b, :, o:o + Tw], xw[b]), b
        assert torch.equal(so[b, :, o:o + Tw], skw[b]), b
        assert not xo[b, :, :o].any() and not xo[b, :, o + Tw:].any(), b


@pytest.mark.parametrize("scale,sched", [(4, [1]), (4, [3, 1, 7]), (8, [50])])
def test_masked_fir_stream_bit_for_bit(dev, scale, sched):
    """pwgb_upsample_fir_stream_ext_forward chunked and flushed equals pwgb_upsample_fir_forward on the whole signal, one
    frame later, with zeros outside the signal"""
    from parallelwavegan_b200 import ops

    B, Cc, F = 2, 80, 23
    g = torch.Generator(device=dev).manual_seed(scale * 100 + len(sched))
    x = torch.randn((B, Cc, F), device=dev, generator=g)
    fir = torch.randn(2 * scale + 1, device=dev, generator=g)
    ref = ops.upsample_fir(x, fir, scale)
    hist = torch.zeros((B, Cc, 2), device=dev)
    frame = torch.zeros(B, device=dev, dtype=torch.int32)
    end = torch.full((B,), 2 ** 31 - 1, device=dev, dtype=torch.int32)
    outs, j, k = [], 0, 0
    while j <= F:
        n = 1 if j == F else min(sched[k % len(sched)], F - j)
        if j == F:
            end.fill_(F)
        xi = x[:, :, j:j + n].contiguous() if j < F else torch.zeros((B, Cc, 1), device=dev)
        outs.append(ops.upsample_fir_causal_stream(xi, fir, scale, hist, mask=(frame, end, scale, scale)))
        ops.stream_carry(ops.stream_carry_table([(xi, hist)], dev))
        frame += n
        j, k = j + n, k + 1
    y = torch.cat(outs, -1)
    assert not y[:, :, :scale].any()
    assert torch.equal(y[:, :, scale:], ref)


# ------------------------------------------------------------------------------------------------ slots, reset, graphs
def test_batch_slots_are_independent(dev):
    from parallelwavegan_b200.streaming import PWGLookaheadStream

    m = _model(dev)
    c, z = _inputs(m, 4, 30, 430)
    st = PWGLookaheadStream(m, batch=4, use_graphs=False)
    ref = _expected(m, c, z, st.delay)
    y = _stream(st, c.to(dev), z.to(dev), SCHEDULES["mixed"], m.upsample_factor)
    st1 = PWGLookaheadStream(m, batch=1, use_graphs=False)
    for b in range(4):
        assert torch.equal(y[b], ref[b]), b
        assert torch.equal(_stream(st1, c[b:b + 1].to(dev), z[b:b + 1].to(dev), [5], m.upsample_factor)[0], y[b]), b


def test_state_bytes(dev):
    """fp32 conv_in, FIR, noise, conditioning and skip histories, (K-1)*d packed hi/lo bf16 rows of R channels per WaveNet
    layer and the two int32 frame counters"""
    from parallelwavegan_b200.streaming import PWGLookaheadStream

    m = _model(dev)
    st = PWGLookaheadStream(m, batch=3)
    A, R, S = 80, 64, 64
    W = 3069 - 1  # conditioning rows and skip columns kept: the last layer's lag behind layer 0
    wn = sum(R * 2 * f.dilation for f in m.conv_layers)
    assert st.state_bytes() == 4 * (A * 4 + 2 * A * 4 + 851 + A * W + S * W + wn + 2)
    assert 3.2e6 < st.state_bytes() < 3.4e6


def test_reset_and_flush_keep_other_slots(dev):
    """a mid-stream reset of slot 0 and a flush of slot 0 while slot 1 streams on: slot 1 is bit-identical to an
    uninterrupted run, and slot 0's restarted utterances are bit-identical to inference"""
    from parallelwavegan_b200.streaming import PWGLookaheadStream

    m = _model(dev)
    hop = m.upsample_factor
    c, z = _inputs(m, 2, 36, 440)
    st = PWGLookaheadStream(m, batch=2, use_graphs=True)
    ref1 = _stream(PWGLookaheadStream(m, batch=2, use_graphs=True), c.to(dev), z.to(dev), [3], hop)[1]
    cd, zd = c.to(dev), z.to(dev)
    outs1, seg = [], []
    for j in range(0, 36, 3):
        if j == 9:
            st.reset(0)  # slot 0 restarts at frame 9
            seg = []
        if j == 24:
            tail = st.flush(0)  # slot 0's utterance (frames 9 .. 23) ends; slot 1 carries on
            seg.append(tail[0])
            exp = _expected(m, c[:1, 9:24], z[:1, :, 9 * hop:24 * hop], st.delay)[0]
            assert torch.equal(torch.cat(seg, -1), exp)
        y = st.push(cd[:, j:j + 3], zd[:, :, j * hop:(j + 3) * hop])
        outs1.append(y[1])
        seg.append(y[0])
    outs1.append(st.flush(1)[0])
    assert torch.equal(torch.cat(outs1, -1), ref1)


def test_graphs_replay_eager_and_many_chunk_lengths(dev):
    """more distinct chunk lengths than MAX_CHUNK_LENGTHS: the entry cache is rebuilt and graphs recaptured"""
    from parallelwavegan_b200.streaming import PWGLookaheadStream

    m = _model(dev)
    sched = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 1, 3]
    assert len(set(sched)) > PWGLookaheadStream.MAX_CHUNK_LENGTHS
    c, z = _inputs(m, 2, 69, 450)
    g = _stream(PWGLookaheadStream(m, batch=2, use_graphs=True), c.to(dev), z.to(dev), sched, m.upsample_factor)
    e = _stream(PWGLookaheadStream(m, batch=2, use_graphs=False), c.to(dev), z.to(dev), sched, m.upsample_factor)
    assert torch.equal(g, e)
    assert torch.equal(g, _expected(m, c, z, 3920).to(dev))


def test_unsupported_models_raise(dev):
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import PWGLookaheadStream

    cases = [dict(use_causal_conv=True), dict(upsample_net="MelGANGenerator", aux_context_window=0,
                                               upsample_params={"upsample_scales": [4, 4, 4, 4]}),
             dict(upsample_conditional_features=False), dict(residual_channels=8, gate_channels=16, skip_channels=8, aux_channels=10)]
    for over in cases:
        with pytest.raises(PwgbError):
            PWGLookaheadStream(_model(dev, **over))
    m, _, _, _ = _golden_model(dev, "pwg_small")  # 8 residual, 10 aux channels: outside the fused stack
    with pytest.raises(PwgbError):
        PWGLookaheadStream(m)
    m = _model(dev)
    with pytest.raises(PwgbError):
        PWGLookaheadStream(m.cpu())
    m = _model(dev).train()
    with pytest.raises(PwgbError):
        PWGLookaheadStream(m)
    with pytest.raises(PwgbError, match="CausalPWGStream"):
        PWGLookaheadStream(_model(dev, use_causal_conv=True))
