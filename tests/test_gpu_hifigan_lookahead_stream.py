"""Streaming the centred HiFi-GAN on the GPU (parallelwavegan_b200.streaming.HiFiGANLookaheadStream): the extended history
conv entry points (mask, delayed residual, delayed read) and the masked conv-transpose are bit-identical to the existing
entry points on the explicit signal, streamed audio followed by the flush is bit-identical to
[zeros(delay) | inference] for every chunk schedule, slots are independent (also across a flush), graphs replay what
eager runs compute, and the unsupported models raise."""
import json

import pytest
import torch

from helpers import REL_TOL, golden_weights, load_golden, rel_l2
from oracle import synth
from stream_harness import dev, debug_get, KCASES, mels  # noqa: F401

pytestmark = pytest.mark.gpu

# one frame at a time, 3 frames, longer than the input conv's 6-frame history, and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
V1 = dict(in_channels=80, out_channels=1, channels=512, kernel_size=7, upsample_scales=[8, 8, 2, 2],
          upsample_kernel_sizes=[16, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3,
          use_causal_conv=False)
# whole utterances up to 15 frames: the output conv takes the generic FFMA kernel on both sides (DESIGN.md)
FRAMES = 15
GOLDEN = ["hifigan_small", "hifigan_odd", "hifigan_v1"]


def _golden(dev, name, weight_norm=True):
    from parallelwavegan_b200 import models

    meta, g = load_golden(name)
    m = models.HiFiGANGenerator(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    if not weight_norm:
        m.remove_weight_norm()
    return meta, g, m.to(dev).eval()


def _model(dev, name, weight_norm=True):
    if name != "v1_512":
        return _golden(dev, name, weight_norm)[2]
    from parallelwavegan_b200 import models

    m = models.HiFiGANGenerator(**json.loads(json.dumps(V1)))
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 7, 1.15))
    if not weight_norm:
        m.remove_weight_norm()
    return m.to(dev).eval()


def _stream(st, c, schedule, flush=True):
    """c: (B, T, in_channels) pushed in chunks of ``schedule`` frames, then flushed; the concatenated output"""
    outs, j, k = [], 0, 0
    while j < c.shape[1]:
        n = min(schedule[k % len(schedule)], c.shape[1] - j)
        outs.append(st.push(c[:, j:j + n]))
        j, k = j + n, k + 1
    if flush:
        outs.append(st.flush())
    return torch.cat(outs, -1)


def _expected(m, c, delay):
    """[zeros(delay) | model.inference] of each item alone: (B, out_channels, delay + T * hop)"""
    d = next(m.parameters()).device
    with torch.no_grad():
        y = torch.stack([m.inference(c[b].to(d)).t() for b in range(c.shape[0])])
    return torch.cat([y.new_zeros(y.shape[:-1] + (delay,)), y], -1)


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("name", list(KCASES))
def test_conv_stream_ext_bit_exact(dev, name):
    """mask, delayed residual and delayed read against the existing entry point on the explicit [hist | x], masked
    afterwards"""
    from parallelwavegan_b200 import ops

    B, cin, cout, K, d, n, H, pl, rep, epi, engine, plan = KCASES[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)) + 1)
    delta = 2  # the delayed read: rows [-(pad_left + delta), t_out - delta) (every case has H <= pad_left)
    x = torch.randn(B, cin, n, generator=g).to(dev)
    hist = torch.randn(B, cin, H, generator=g).to(dev)
    w = (torch.randn(cout, cin, K, generator=g) / (cin * K) ** 0.5).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    t_out = n + pl - d * (K - 1)
    Hr, rd = 9, 5
    r = torch.randn(B, cout, t_out, generator=g).to(dev)
    rh = torch.randn(B, cout, Hr, generator=g).to(dev)
    y0 = torch.randn(B, cout, t_out, generator=g).to(dev)
    # slot frames and ends: one slot at its start, one ended inside the chunk, the others open
    rate, look = 3, 7
    frame = torch.tensor([0, 4, 1][:B] + [2] * max(B - 3, 0), dtype=torch.int32, device=dev)
    end = torch.full((B,), 2 ** 31 - 1, dtype=torch.int32, device=dev)
    if B > 1:
        end[1] = frame[1] + (t_out // 2 + look) // rate
    kw = dict(pre_slope=0.1)
    residual = epi in ("res", "acc")
    if epi == "res":
        kw.update(out_scale=0.5)
    elif epi == "tanh":
        kw.update(pre_slope=0.01, post_act="tanh")
    repl = torch.tensor(rep, dtype=torch.int32, device=dev) if rep is not None else None
    h_eff = hist.clone()
    for i, f in enumerate(rep or []):
        if f:
            h_eff[i] = x[i, :, :1].expand(-1, H)
    xc = torch.cat([h_eff, x], -1)
    r_eff = torch.cat([rh, r], -1)[..., Hr - rd:Hr - rd + t_out].contiguous()
    pos = frame[:, None, None].long() * rate - look + torch.arange(t_out, device=dev)
    inside = (pos >= 0) & (pos < end[:, None, None].long() * rate)
    old = ops.ENGINE
    ops.ENGINE = "simt" if engine == "simt" else "auto"
    try:
        outs = []
        for stream in (True, False):
            o = y0.clone() if epi == "acc" else None
            extra = dict(out=o, accumulate=True, out_scale=1 / 3) if epi == "acc" else {}
            if stream:
                res = dict(residual=r, res_hist=rh, res_delay=rd) if residual else {}
                y = ops.conv1d_stream(x, hist, w, b, pad_left=pl + delta, dilation=d, replicate=repl, t_out=t_out,
                                      mask=(frame, end, rate, look), **res, **kw, **extra)
                if engine == "tc":
                    p = debug_get(1, 8)
                    assert p[5] == 0 and p[4] == 0, p  # no TMA activation rows, the register epilogue
                else:
                    assert debug_get(3, 6)[0] == 0
            else:
                # the explicit conv computes delta more rows; the residual and the accumulated output are padded to them
                pad = lambda t: torch.nn.functional.pad(t, (0, delta))  # noqa: E731
                if epi == "acc":
                    extra["out"] = pad(o)
                y = ops.conv1d_raw(xc, w, b, dilation=d, padding=(pl + delta - H, 0), **kw, **extra,
                                   **(dict(residual=pad(r_eff)) if residual else {}))
                y = torch.where(inside, y[..., :t_out], torch.zeros((), device=dev))
            outs.append(y)
    finally:
        ops.ENGINE = old
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("engine", ["tc", "simt"])
def test_conv_transpose_stream_equals_whole_signal(dev, engine):
    """the masked stream conv-transpose with the centred layer's padding, chunk by chunk and then flushed, equals
    pwgb_conv_transpose1d_forward on the whole signal, labelled p samples later"""
    from parallelwavegan_b200 import ops

    cin, cout, s, B, T = (64, 32, 8, 3, 37) if engine == "tc" else (16, 8, 3, 2, 41)
    p = s // 2 + s % 2
    g = torch.Generator().manual_seed(6)
    x = torch.randn(B, cin, T, generator=g).to(dev)
    w = (torch.randn(cin, cout, 2 * s, generator=g) / cin ** 0.5).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    ref = ops.conv_transpose1d_raw(x, w, b, stride=s, padding=p, output_padding=s % 2, pre_slope=0.1)
    frame = torch.zeros(B, dtype=torch.int32, device=dev)
    end = torch.full((B,), 2 ** 31 - 1, dtype=torch.int32, device=dev)
    hist = torch.zeros(B, cin, 1, device=dev)
    old = ops.ENGINE
    ops.ENGINE = "simt" if engine == "simt" else "auto"
    try:
        outs, j = [], 0
        for n in [1, 5, 2, 11, 3] * 10:
            n = min(n, T - j)
            if n == 0:
                break
            chunk = x[:, :, j:j + n].contiguous()
            outs.append(ops.conv_transpose1d_stream(chunk, hist, w, b, stride=s, pre_slope=0.1, mask=(frame, end, s, p)))
            hist = chunk[:, :, -1:].contiguous()
            frame += n
            j += n
        end.copy_(frame)
        outs.append(ops.conv_transpose1d_stream(torch.zeros(B, cin, 2, device=dev), hist, w, b, stride=s, pre_slope=0.1,
                                                mask=(frame, end, s, p)))
    finally:
        ops.ENGINE = old
    y = torch.cat(outs, -1)
    assert torch.equal(y[..., :p], torch.zeros_like(y[..., :p]))
    assert torch.equal(y[..., p:p + T * s], ref)
    assert torch.equal(y[..., p + T * s:], torch.zeros_like(y[..., p + T * s:]))


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("weight_norm", [True, False])
@pytest.mark.parametrize("name", GOLDEN + ["v1_512"])
def test_stream_equals_inference(dev, name, weight_norm, schedule):
    from parallelwavegan_b200.streaming import HiFiGANLookaheadStream

    m = _model(dev, name, weight_norm)
    c = mels(2, FRAMES, 61)
    st = HiFiGANLookaheadStream(m, batch=2)
    ref = _expected(m, c, st.delay)
    assert debug_get(3, 6)[0] == 0  # the output conv of the whole utterance took the generic kernel
    y = _stream(st, c, SCHEDULES[schedule])
    assert debug_get(3, 6)[0] == 0  # and so did the stream's (the flush's, the last FFMA launch)
    assert torch.equal(y, ref)


@pytest.mark.parametrize("frames", [1, 2])
@pytest.mark.parametrize("name", ["hifigan_small", "hifigan_odd", "v1_512"])
def test_short_utterances_come_from_the_flush(dev, name, frames):
    from parallelwavegan_b200.streaming import HiFiGANLookaheadStream

    m = _model(dev, name)
    c = mels(2, frames, 62)
    st = HiFiGANLookaheadStream(m, batch=2)
    assert frames * st.hop < st.delay
    assert torch.equal(_stream(st, c, [1]), _expected(m, c, st.delay))


def test_delay_from_the_module(dev):
    from oracle.ref_hifigan_lookahead_stream import HiFiGANLookaheadRef
    from parallelwavegan_b200.streaming import HiFiGANLookaheadStream

    assert HiFiGANLookaheadStream(_model(dev, "v1_512")).delay == 3258
    meta, _, m = _golden(dev, "hifigan_odd")
    st = HiFiGANLookaheadStream(m)
    assert st.delay == 170
    cfg = dict(meta["kwargs"], negative_slope=0.1)
    assert st.delay == HiFiGANLookaheadRef({k: v.double() for k, v in golden_weights(meta).items()}, cfg).delay


@pytest.mark.parametrize("name", GOLDEN)
def test_stream_matches_reference_output(dev, name):
    from parallelwavegan_b200.streaming import HiFiGANLookaheadStream

    meta, g, m = _golden(dev, name)
    c = synth.randn(meta["c_shape"], meta["c_seed"])[0].t()
    st = HiFiGANLookaheadStream(m)
    y = _stream(st, c[None], SCHEDULES["mixed"])
    assert rel_l2(y[0, :, st.delay:].t().cpu(), g["y_inf"]) < REL_TOL


def test_long_utterance_within_rel_l2(dev):
    """48 frames: the whole utterance's output conv takes conv1d_fewcout_long_kernel, whose sum order a stream cannot
    reproduce"""
    from parallelwavegan_b200.streaming import HiFiGANLookaheadStream

    m = _model(dev, "hifigan_small")
    c = mels(2, 48, 63)
    st = HiFiGANLookaheadStream(m, batch=2)
    ref = _expected(m, c, st.delay)
    assert debug_get(3, 6)[0] == 2
    y = _stream(st, c, SCHEDULES["mixed"])
    assert rel_l2(y.cpu(), ref.cpu()) <= 1e-6


def test_batch_slots_reset_flush_and_graphs(dev):
    """B = 4 equals four B = 1 streams, graph replay equals eager, a mid-stream reset of one slot restarts only that
    slot, and flushing slot 0 leaves slot 1's whole output bit-identical to an uninterrupted run"""
    from parallelwavegan_b200.streaming import HiFiGANLookaheadStream

    m = _model(dev, "v1_512")
    c = mels(4, FRAMES, 64)
    y4 = _stream(HiFiGANLookaheadStream(m, batch=4), c, SCHEDULES["mixed"])
    for b in range(4):
        assert torch.equal(y4[b:b + 1], _stream(HiFiGANLookaheadStream(m, batch=1), c[b:b + 1], SCHEDULES["mixed"]))
    assert torch.equal(_stream(HiFiGANLookaheadStream(m, batch=4, use_graphs=False), c, SCHEDULES["mixed"]), y4)
    # slot 1 restarts after 6 frames on a new utterance; the other slots continue
    st = HiFiGANLookaheadStream(m, batch=4)
    first = _stream(st, c[:, :6], [2, 4], flush=False)
    c2 = c.clone()
    c2[1, 6:] = mels(1, FRAMES - 6, 65)[0]
    st.reset(1)
    rest = _stream(st, c2[:, 6:], [1, 3, 5])
    y = torch.cat([first, rest], -1)
    for b in (0, 2, 3):
        assert torch.equal(y[b], y4[b])
    assert torch.equal(rest[1:2], _expected(m, c2[1:2, 6:], st.delay))
    # slot 0 ends after 5 frames and is flushed while slot 1 keeps streaming
    st = HiFiGANLookaheadStream(m, batch=2)
    a = st.push(c[:2, :5])
    f0 = st.flush(0)
    assert f0.shape == (1, 1, st.delay)
    assert torch.equal(torch.cat([a[:1], f0], -1), _expected(m, c[:1, :5], st.delay))
    rest = _stream(st, c[:2, 5:], [3, 1, 6])
    uninterrupted = _stream(HiFiGANLookaheadStream(m, batch=1), c[1:2], SCHEDULES["mixed"])
    assert torch.equal(torch.cat([a[1:2], rest[1:2]], -1), uninterrupted)
    # slot 0 started over on frames 5.. of its utterance
    assert torch.equal(rest[:1], _expected(m, c[:1, 5:], st.delay))


def test_more_chunk_lengths_than_cached(dev):
    """55 frames of the odd model (hop 30) keep the whole utterance's output conv below 4096 samples, on the generic
    kernel"""
    from parallelwavegan_b200.streaming import HiFiGANLookaheadStream

    m = _model(dev, "hifigan_odd")
    st = HiFiGANLookaheadStream(m, batch=2)
    sched = list(range(1, st.MAX_CHUNK_LENGTHS + 3))
    c = mels(2, sum(sched), 66)
    assert torch.equal(_stream(st, c, sched), _expected(m, c, st.delay))


def test_unsupported_models_raise(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import HiFiGANLookaheadStream

    small = dict(V1, channels=32)
    with pytest.raises(PwgbError, match="CausalHiFiGANStream"):
        HiFiGANLookaheadStream(models.HiFiGANGenerator(**dict(small, use_causal_conv=True)).to(dev).eval())
    with pytest.raises(PwgbError, match="train mode"):
        HiFiGANLookaheadStream(models.HiFiGANGenerator(**small).to(dev).train())
    with pytest.raises(PwgbError, match="CUDA"):
        HiFiGANLookaheadStream(models.HiFiGANGenerator(**small).eval())
    with pytest.raises(PwgbError):
        HiFiGANLookaheadStream(models.HiFiGANGenerator(**small).to(dev).eval(), batch=0)
    for other in (models.UHiFiGANGenerator(), models.DiscreteSymbolHiFiGANGenerator(num_spk_embs=0),
                  models.ParallelWaveGANGenerator(), models.MelGANGenerator()):
        with pytest.raises(PwgbError):
            HiFiGANLookaheadStream(other.to(dev).eval())
