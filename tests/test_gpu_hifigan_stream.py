"""Streaming the causal HiFi-GAN on the GPU (parallelwavegan_b200.streaming.CausalHiFiGANStream): the history conv entry
points, the causal conv-transpose entry and the carry are bit-identical to the existing entry points on the
concatenated signal, streamed audio is bit-identical to ``inference`` on the whole utterance for every chunk schedule,
slots are independent, graphs replay what eager runs compute, and the unsupported models raise."""
import json

import pytest
import torch

from helpers import REL_TOL, golden_weights, load_golden, rel_l2
from oracle import synth
from stream_harness import dev, debug_get, KCASES, mels  # noqa: F401

pytestmark = pytest.mark.gpu

# one frame at a time, 3 frames, longer than the deepest history (the input conv's 6 frames), and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
# HiFi-GAN v1 shapes with synthetic weights: 512 channels, tensor-core convs and the 80 -> 96 padded input conv
V1 = dict(in_channels=80, out_channels=1, channels=512, kernel_size=7, upsample_scales=[8, 8, 2, 2],
          upsample_kernel_sizes=[16, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3,
          use_causal_conv=True)
# whole utterances up to 15 frames: every few-channel conv takes the generic FFMA kernel on both sides (DESIGN.md)
FRAMES = 15


def _golden(dev, weight_norm=True):
    from parallelwavegan_b200 import models

    meta, g = load_golden("hifigan_causal")
    m = models.HiFiGANGenerator(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    if not weight_norm:
        m.remove_weight_norm()
    return meta, g, m.to(dev).eval()


def _v1(dev, weight_norm=True, **over):
    from parallelwavegan_b200 import models

    m = models.HiFiGANGenerator(**json.loads(json.dumps(dict(V1, **over))))
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 7, 1.15))
    if not weight_norm:
        m.remove_weight_norm()
    return m.to(dev).eval()


def _stream(st, c, schedule):
    """c: (B, T, in_channels) pushed in chunks of ``schedule`` frames; the concatenated output"""
    outs, j, k = [], 0, 0
    while j < c.shape[1]:
        n = min(schedule[k % len(schedule)], c.shape[1] - j)
        outs.append(st.push(c[:, j:j + n]))
        j, k = j + n, k + 1
    return torch.cat(outs, -1)


def _inference(m, c):
    """model.inference of each item alone: (B, out_channels, T * hop)"""
    d = next(m.parameters()).device
    with torch.no_grad():
        return torch.stack([m.inference(c[b].to(d)).t() for b in range(c.shape[0])])


# ---------------------------------------------------------------------------------------------------- kernels


@pytest.mark.parametrize("name", list(KCASES))
def test_conv_stream_bit_exact(dev, name):
    from parallelwavegan_b200 import ops

    B, cin, cout, K, d, n, H, pl, rep, epi, engine, plan = KCASES[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(B, cin, n, generator=g).to(dev)
    hist = torch.randn(B, cin, H, generator=g).to(dev)
    w = (torch.randn(cout, cin, K, generator=g) / (cin * K) ** 0.5).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    t_out = n + pl - d * (K - 1)
    r = torch.randn(B, cout, t_out, generator=g).to(dev)
    y0 = torch.randn(B, cout, t_out, generator=g).to(dev)
    kw = dict(pre_slope=0.1)
    if epi == "res":
        kw.update(residual=r, out_scale=0.5)
    elif epi == "tanh":
        kw.update(pre_slope=0.01, post_act="tanh")
    repl = torch.tensor(rep, dtype=torch.int32, device=dev) if rep is not None else None
    h_eff = hist.clone()
    for i, f in enumerate(rep or []):
        if f:
            h_eff[i] = x[i, :, :1].expand(-1, H)
    xc = torch.cat([h_eff, x], -1)
    old = ops.ENGINE
    ops.ENGINE = "simt" if engine == "simt" else "auto"
    try:
        outs = []
        for stream in (True, False):
            o = y0.clone() if epi == "acc" else None
            extra = dict(out=o, accumulate=True, out_scale=1 / 3) if epi == "acc" else {}
            if stream:
                y = ops.conv1d_stream(x, hist, w, b, pad_left=pl, dilation=d, replicate=repl, **kw, **extra)
                if engine == "tc":
                    p = debug_get(1, 8)
                    assert p[5] == 0, p  # no TMA activation rows in a history launch
                    assert {"cp": p[3] > 0 and not p[6], "direct": p[3] == 0, "win": p[6] == 1, "nco": p[7] > 1}[plan], p
                else:
                    assert debug_get(3, 6)[0] == 0
            else:
                y = ops.conv1d_raw(xc, w, b, dilation=d, padding=(pl - H, 0), **kw, **extra)
                if engine == "simt":
                    assert debug_get(3, 6)[0] == 0
            outs.append(y)
    finally:
        ops.ENGINE = old
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("engine", ["tc", "simt"])
def test_conv_transpose_stream_bit_exact(dev, engine):
    from parallelwavegan_b200 import ops

    cin, cout, s, B, n = (64, 32, 8, 3, 37) if engine == "tc" else (16, 8, 2, 3, 41)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, cin, n, generator=g).to(dev)
    hist = torch.randn(B, cin, 1, generator=g).to(dev)
    w = (torch.randn(cin, cout, 2 * s, generator=g) / cin ** 0.5).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    rep = torch.tensor([1, 0, 1], dtype=torch.int32, device=dev)
    y = ops.conv_transpose1d_stream(x, hist, w, b, stride=s, replicate=rep, pre_slope=0.1)
    h = torch.where(rep.bool()[:, None, None], x[:, :, :1], hist)
    ref = ops.conv_transpose1d_raw(torch.cat([h, x], -1), w, b, stride=s, padding=s, pre_slope=0.1)
    assert torch.equal(y, ref)


def test_stream_carry_matches_slicing(dev):
    from parallelwavegan_b200 import ops

    g = torch.Generator().manual_seed(9)
    shapes = [(3, 5, 2, 7), (2, 64, 40, 10), (1, 3, 9, 0), (4, 8, 300, 300), (2, 16, 1, 1), (3, 2, 5, 600)] * 4  # (B, C, n, H)
    ents, refs = [], []
    for B, Cc, n, H in shapes:
        x = torch.randn(B, Cc, n, generator=g).to(dev)
        h = torch.randn(B, Cc, H, generator=g).to(dev)
        refs.append(torch.cat([h, x], -1)[..., -H:] if H else h.clone())
        ents.append((x, h))
    ops.stream_carry(ops.stream_carry_table(ents, dev))
    for (_, h), ref in zip(ents, refs):
        assert torch.equal(h, ref)


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("weight_norm", [True, False])
def test_golden_stream_equals_inference(dev, weight_norm, schedule):
    from parallelwavegan_b200.streaming import CausalHiFiGANStream

    meta, _, m = _golden(dev, weight_norm)
    c = synth.randn(meta["c_shape"], meta["c_seed"]).transpose(1, 2)[:, :FRAMES].contiguous()
    ref = _inference(m, c)
    assert debug_get(3, 6)[0] == 0  # the output conv of the whole utterance took the generic kernel
    y = _stream(CausalHiFiGANStream(m, batch=c.shape[0]), c, SCHEDULES[schedule])
    assert torch.equal(y, ref)


def test_golden_stream_matches_reference_output(dev):
    from parallelwavegan_b200.streaming import CausalHiFiGANStream

    meta, g, m = _golden(dev)
    c = synth.randn(meta["c_shape"], meta["c_seed"])[0].t()
    y = _stream(CausalHiFiGANStream(m), c[None], SCHEDULES["mixed"])
    assert rel_l2(y[0].t().cpu(), g["y_inf"]) < REL_TOL


def test_long_utterance_within_rel_l2(dev):
    """48 frames: the whole utterance's few-channel convs take conv1d_fewcout_long_kernel, whose sum order a stream cannot
    reproduce"""
    from parallelwavegan_b200.streaming import CausalHiFiGANStream

    _, _, m = _golden(dev)
    c = mels(2, 48, 31)
    ref = _inference(m, c)
    y = _stream(CausalHiFiGANStream(m, batch=2), c, SCHEDULES["mixed"])
    assert rel_l2(y.cpu(), ref.cpu()) <= 1e-6


@pytest.mark.parametrize("variant", ["wn", "plain", "no_additional_convs"])
@pytest.mark.parametrize("schedule", ["ones", "long", "mixed"])
def test_v1_stream_equals_inference(dev, variant, schedule):
    from parallelwavegan_b200.streaming import CausalHiFiGANStream

    m = _v1(dev, weight_norm=variant == "wn", **({"use_additional_convs": False} if variant == "no_additional_convs" else {}))
    c = mels(1, FRAMES, 41)
    ref = _inference(m, c)
    y = _stream(CausalHiFiGANStream(m), c, SCHEDULES[schedule])
    assert torch.equal(y, ref)


def test_batch_slots_reset_and_graphs(dev):
    """B = 4 equals four B = 1 streams, a mid-stream reset of one slot restarts only that slot, and graph replay equals
    eager"""
    from parallelwavegan_b200.streaming import CausalHiFiGANStream

    m = _v1(dev)
    c = mels(4, FRAMES, 51)
    y4 = _stream(CausalHiFiGANStream(m, batch=4), c, SCHEDULES["mixed"])
    for b in range(4):
        assert torch.equal(y4[b:b + 1], _stream(CausalHiFiGANStream(m, batch=1), c[b:b + 1], SCHEDULES["mixed"]))
    assert torch.equal(_stream(CausalHiFiGANStream(m, batch=4, use_graphs=False), c, SCHEDULES["mixed"]), y4)
    # slot 1 restarts after 6 frames on a new utterance; the other slots continue
    st = CausalHiFiGANStream(m, batch=4)
    first = _stream(st, c[:, :6], [2, 4])
    c2 = c.clone()
    c2[1, 6:] = mels(1, FRAMES - 6, 52)[0]
    st.reset(1)
    rest = _stream(st, c2[:, 6:], [1, 3, 5])
    y = torch.cat([first, rest], -1)
    hop = y.shape[-1] // FRAMES
    for b in (0, 2, 3):
        assert torch.equal(y[b], y4[b])
    assert torch.equal(rest[1:2], _inference(m, c2[1:2, 6:]))
    assert torch.equal(first[1], y4[1, :, :6 * hop])


def test_unsupported_models_raise(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import CausalHiFiGANStream

    small = dict(V1, channels=32)
    with pytest.raises(PwgbError):
        CausalHiFiGANStream(models.HiFiGANGenerator(**dict(small, use_causal_conv=False)).to(dev).eval())
    with pytest.raises(PwgbError):
        CausalHiFiGANStream(models.HiFiGANGenerator(**small).to(dev).train())
    with pytest.raises(PwgbError):
        CausalHiFiGANStream(models.HiFiGANGenerator(**small).eval())
    with pytest.raises(PwgbError):
        CausalHiFiGANStream(models.HiFiGANGenerator(**small).to(dev).eval(), batch=0)
    for other in (models.UHiFiGANGenerator(), models.DiscreteSymbolHiFiGANGenerator(num_spk_embs=0),
                  models.ParallelWaveGANGenerator(use_causal_conv=True)):
        with pytest.raises(PwgbError):
            CausalHiFiGANStream(other.to(dev).eval())
