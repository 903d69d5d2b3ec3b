"""Streaming the causal (multi-band) MelGAN on the GPU (parallelwavegan_b200.streaming.CausalMelGANStream): the
reflect-flag history convs are bit-identical to the reflect-padded whole-signal convs on every engine and plan, the
synthesis window is bit-identical to ``PQMF.synthesis``, streamed audio plus flush is bit-identical to ``inference``
after the PQMF delay for every pad and chunk schedule, slots are independent, graphs replay what eager runs compute, and
the unsupported cases raise."""
import json

import pytest
import torch
import torch.nn.functional as F

from helpers import REL_TOL, golden_weights, load_golden, rel_l2
from oracle import synth
from stream_harness import dev, debug_get, mels  # noqa: F401

pytestmark = pytest.mark.gpu

# after an opening push of min_first_frames: one frame at a time, 3 frames, and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "mixed": [1, 4, 2, 9, 1, 3]}
# MelGAN v1 (egs/ljspeech/voc1/conf/melgan.v1.long.yaml) and multi-band MelGAN v2 shapes with synthetic weights
V1 = dict(in_channels=80, out_channels=1, kernel_size=7, channels=512, upsample_scales=[8, 8, 2, 2], stack_kernel_size=3, stacks=3,
          use_causal_conv=True)
MB2 = dict(in_channels=80, out_channels=4, kernel_size=7, channels=384, upsample_scales=[8, 4, 2], stack_kernel_size=3, stacks=4,
           use_causal_conv=True)
# whole utterances below 4096 output-conv samples (15 frames of v1, 63 of MB v2): every few-channel conv takes the
# generic FFMA kernel on both sides (DESIGN.md section 3.7)
FRAMES = {"v1": 15, "mb2": 40}
GOLDEN = ["melgan_causal", "melgan_causal_replicate", "melgan_causal_zero", "melgan_causal_mb"]


def _golden(dev, name, weight_norm=True):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.layers import PQMF

    meta, g = load_golden(name)
    m = models.MelGANGenerator(**json.loads(json.dumps(meta["kwargs"])))
    m.load_state_dict(golden_weights(meta), strict=True)
    if not weight_norm:
        m.remove_weight_norm()
    m = m.to(dev).eval()
    if meta.get("pqmf_subbands"):
        m.pqmf = PQMF(meta["pqmf_subbands"]).to(dev)
    return meta, g, m


def _synthetic(dev, kind, weight_norm=True, **over):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.layers import PQMF

    kw = dict(V1 if kind == "v1" else MB2, **over)
    m = models.MelGANGenerator(**json.loads(json.dumps(kw)))
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 8, 1.0))
    if not weight_norm:
        m.remove_weight_norm()
    m = m.to(dev).eval()
    if kind == "mb2":
        m.pqmf = PQMF(4).to(dev)
    return m


def _stream(st, c, schedule, first=None, flush=True):
    """c: (B, T, in_channels) pushed as ``first`` frames (default: min_first_frames), then chunks of ``schedule``
    frames; the concatenated output, with the flush"""
    first = st.min_first_frames if first is None else first
    outs, j, k = [st.push(c[:, :first])], first, 0
    while j < c.shape[1]:
        n = min(schedule[k % len(schedule)], c.shape[1] - j)
        outs.append(st.push(c[:, j:j + n]))
        j, k = j + n, k + 1
    if flush:
        outs.append(st.flush())
    return torch.cat(outs, -1)


def _inference(m, c, delay=0):
    """[zeros(delay) | model.inference] of each item alone: (B, 1, delay + T * hop * subbands)"""
    d = next(m.parameters()).device
    with torch.no_grad():
        y = torch.stack([m.inference(c[b].to(d)).t() for b in range(c.shape[0])])
    return F.pad(y, (delay, 0))


# ---------------------------------------------------------------------------------------------------- kernels
# name: B, cin, cout, K, dilation, n, pad_left (== H), fresh flags, epilogue, engine, expected plan
#   plan (tensor cores, pwgb_debug_get(1)): "cp" cp.async-staged, "direct" register path, "win" win_mode, "nco" column chunks
KCASES = {
    "tc_cp": (2, 64, 64, 3, 2, 300, 4, [1, 0], "plain", "tc", "cp"),
    "tc_cp_all": (3, 96, 48, 7, 1, 200, 6, [1, 1, 1], "res", "tc", "cp"),
    "tc_direct": (2, 32, 32, 3, 176, 400, 352, [0, 1], "plain", "tc", "direct"),
    "tc_win": (1, 32, 32, 3, 1100, 2300, 2200, [1], "plain", "tc", "win"),
    "tc_nco_staged": (3, 32, 256, 11, 5, 700, 50, [1, 0, 0], "res", "tc", "nco"),
    "ffma": (2, 16, 8, 3, 3, 257, 6, [0, 1], "plain", "simt", None),
    "ffma_res": (3, 8, 2, 7, 1, 90, 6, [1, 0, 1], "res", "simt", None),
    "ffma_tanh": (3, 32, 1, 7, 1, 3000, 6, [0, 1, 1], "tanh", "simt", None),
}


@pytest.mark.parametrize("name", list(KCASES))
def test_reflect_conv_stream_bit_exact(dev, name):
    """flagged slots equal the whole-signal conv with left reflect padding, the others the conv on [history | x]"""
    from parallelwavegan_b200 import ops

    B, cin, cout, K, d, n, pl, flags, epi, engine, plan = KCASES[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    x = torch.randn(B, cin, n, generator=g).to(dev)
    hist = torch.randn(B, cin, pl, generator=g).to(dev)
    w = (torch.randn(cout, cin, K, generator=g) / (cin * K) ** 0.5).to(dev)
    b = torch.randn(cout, generator=g).to(dev)
    r = torch.randn(B, cout, n, generator=g).to(dev)
    kw = dict(pre_slope=0.2)
    if epi == "res":
        kw.update(residual=r, out_scale=0.5)
    elif epi == "tanh":
        kw.update(pre_slope=0.01, post_act="tanh")
    fresh = torch.tensor(flags, dtype=torch.int32, device=dev)
    old = ops.ENGINE
    ops.ENGINE = "simt" if engine == "simt" else "auto"
    try:
        y = ops.conv1d_stream(x, hist, w, b, pad_left=pl, dilation=d, replicate=fresh, reflect=True, **kw)
        if engine == "tc":
            p = debug_get(1, 8)
            assert p[5] == 0, p  # no TMA activation rows in a history launch
            assert {"cp": p[3] > 0 and not p[6], "direct": p[3] == 0, "win": p[6] == 1, "nco": p[7] > 1}[plan], p
        else:
            assert debug_get(3, 6)[0] == 0
        ref_reflect = ops.conv1d_raw(x, w, b, dilation=d, padding=(pl, 0), pad_mode="reflect", **kw)
        ref_hist = ops.conv1d_raw(torch.cat([hist, x], -1), w, b, dilation=d, padding=(0, 0), **kw)
    finally:
        ops.ENGINE = old
    for i, f in enumerate(flags):
        assert torch.equal(y[i], (ref_reflect if f else ref_hist)[i]), i


def test_reflect_needs_the_padding_inside_the_chunk(dev):
    from parallelwavegan_b200 import ops
    from parallelwavegan_b200.capi import PwgbError

    x = torch.randn(1, 16, 6, device=dev)
    w = torch.randn(16, 16, 7, device=dev)
    fresh = torch.ones(1, dtype=torch.int32, device=dev)
    with pytest.raises(PwgbError):
        ops.conv1d_stream(x, torch.zeros(1, 16, 6, device=dev), w, pad_left=6, replicate=fresh, reflect=True)


def test_synthesis_window_equals_pqmf_synthesis(dev):
    """slots 0 and 2 start a signal, slot 1 continues one whose first 30 subband samples are its history; chunks of
    several lengths, then the flush"""
    from parallelwavegan_b200 import ops
    from parallelwavegan_b200.layers import PQMF

    pq = PQMF(4).to(dev)
    S = synth.randn((3, 4, 80), 61).to(dev)
    w = (pq.synthesis_filter[0].flip(-1) * 4.0).unsqueeze(1).contiguous()
    whole_fresh = pq.synthesis(S[:, :, 30:].contiguous())
    assert debug_get(3, 6)[0] == 0  # the whole-signal synthesis took the generic FFMA kernel
    whole_cont = pq.synthesis(S)
    fresh = torch.tensor([1, 0, 1], dtype=torch.int32, device=dev)
    hist = torch.zeros(3, 4, 15, device=dev)
    hist[1] = S[1, :, 15:30]
    outs, j = [], 30
    for n in (9, 1, 13, 27):  # a fresh slot's first window covers the 31 samples before 0
        x = S[:, :, j:j + n].contiguous()
        outs.append(ops.conv_transpose1d_window_stream(x, hist, w, None, stride=4, padding=31, fresh=fresh))
        full = torch.cat([hist, x], -1)
        hist = full[:, :, -15:].contiguous()
        fresh = torch.zeros_like(fresh)
        j += n
    outs.append(ops.conv_transpose1d_window_stream(None, hist, w, None, stride=4, padding=31, fresh=fresh, flush_rows=8)[:, :, :31])
    y = torch.cat(outs, -1)
    for b in (0, 2):
        assert torch.equal(y[b], F.pad(whole_fresh[b], (31, 0)))
    assert torch.equal(y[1], whole_cont[1, :, 120 - 31:])
    # a slot flushed before any push holds only the zeros before sample 0
    z = ops.conv_transpose1d_window_stream(None, torch.zeros(1, 4, 15, device=dev), w, None, stride=4, padding=31,
                                           fresh=torch.ones(1, dtype=torch.int32, device=dev), flush_rows=8)
    assert torch.equal(z, torch.zeros_like(z))


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("weight_norm", [True, False])
@pytest.mark.parametrize("name", GOLDEN)
def test_golden_stream_equals_inference(dev, name, weight_norm, schedule):
    from parallelwavegan_b200.streaming import CausalMelGANStream

    meta, _, m = _golden(dev, name, weight_norm)
    c = synth.randn(meta["c_shape"], meta["c_seed"]).transpose(1, 2).contiguous()
    st = CausalMelGANStream(m, batch=c.shape[0])
    assert st.min_first_frames == (7 if name != "melgan_causal_replicate" and name != "melgan_causal_zero" else 1)
    ref = _inference(m, c, st.delay)
    assert debug_get(3, 6)[0] == 0  # the last few-channel conv of the whole utterance took the generic kernel
    assert torch.equal(_stream(st, c, SCHEDULES[schedule]), ref)


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_stream_matches_reference_output(dev, name):
    from parallelwavegan_b200.streaming import CausalMelGANStream

    meta, g, m = _golden(dev, name)
    c = synth.randn(meta["c_shape"], meta["c_seed"])[0].t()
    st = CausalMelGANStream(m)
    y = _stream(st, c[None], SCHEDULES["mixed"])[0, :, st.delay:]
    assert rel_l2(y.t().cpu(), g["y_inf"] if "y_inf" in g else g["y"][0].t()) < REL_TOL


@pytest.mark.parametrize("schedule", ["ones", "mixed"])
@pytest.mark.parametrize("weight_norm", [True, False])
@pytest.mark.parametrize("kind", ["v1", "mb2"])
def test_recipe_shaped_stream_equals_inference(dev, kind, weight_norm, schedule):
    from parallelwavegan_b200.streaming import CausalMelGANStream

    m = _synthetic(dev, kind, weight_norm)
    c = mels(1, FRAMES[kind], 41)
    st = CausalMelGANStream(m)
    assert st.min_first_frames == 7 and st.delay == (31 if kind == "mb2" else 0)
    assert torch.equal(_stream(st, c, SCHEDULES[schedule]), _inference(m, c, st.delay))


@pytest.mark.parametrize("pad", ["replicate", "zero"])
def test_mb_pads_stream_equals_inference(dev, pad):
    from parallelwavegan_b200.streaming import CausalMelGANStream

    over = dict(pad="ReplicationPad1d") if pad == "replicate" else dict(pad="ConstantPad1d", pad_params={"value": 0.0})
    m = _synthetic(dev, "mb2", **over)
    c = mels(2, 20, 43)
    st = CausalMelGANStream(m, batch=2)
    assert st.min_first_frames == 1
    assert torch.equal(_stream(st, c, SCHEDULES["mixed"]), _inference(m, c, st.delay))


@pytest.mark.parametrize("kind", ["golden", "mb2"])
def test_long_utterance_within_rel_l2(dev, kind):
    """past 4096 output-conv samples the whole utterance's few-channel output conv takes conv1d_fewcout_long_kernel, whose
    sum order a stream cannot reproduce"""
    from parallelwavegan_b200.streaming import CausalMelGANStream

    m = _golden(dev, "melgan_causal")[2] if kind == "golden" else _synthetic(dev, "mb2")
    c = mels(2, 300 if kind == "golden" else 80, 31)
    st = CausalMelGANStream(m, batch=2)
    ref = _inference(m, c, st.delay)
    y = _stream(st, c, [5, 16, 3])
    assert rel_l2(y.cpu(), ref.cpu()) <= 1e-6


def test_batch_slots_reset_and_graphs(dev):
    """B = 4 equals four B = 1 streams, a mid-stream reset of one slot restarts only that slot, and graph replay equals
    eager"""
    from parallelwavegan_b200.streaming import CausalMelGANStream

    m = _synthetic(dev, "mb2")
    T = 24
    c = mels(4, T, 51)
    y4 = _stream(CausalMelGANStream(m, batch=4), c, SCHEDULES["mixed"])
    for b in range(4):
        assert torch.equal(y4[b:b + 1], _stream(CausalMelGANStream(m, batch=1), c[b:b + 1], SCHEDULES["mixed"]))
    assert torch.equal(_stream(CausalMelGANStream(m, batch=4, use_graphs=False), c, SCHEDULES["mixed"]), y4)
    # slot 1 is flushed after 10 frames and restarts on a new utterance; the other slots continue
    st = CausalMelGANStream(m, batch=4)
    first = _stream(st, c[:, :10], [3], flush=False)
    tail1 = st.flush(1)
    c2 = c.clone()
    c2[1, 10:] = mels(1, T - 10, 52)[0]
    rest = _stream(st, c2[:, 10:], [1, 3, 5], flush=False)
    end = st.flush()
    y = torch.cat([first, rest, end], -1)
    for b in (0, 2, 3):
        assert torch.equal(y[b], y4[b])
    ref1 = _inference(m, c[1:2, :10], st.delay)
    assert torch.equal(torch.cat([first[1:2], tail1], -1), ref1)
    assert torch.equal(torch.cat([rest[1:2], end[1:2]], -1), _inference(m, c2[1:2, 10:], st.delay))
    assert st.state_bytes() > 0


def test_unsupported_cases_raise(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import CausalMelGANStream

    small = dict(V1, channels=32, upsample_scales=[4, 4], stacks=2)
    st = CausalMelGANStream(models.MelGANGenerator(**small).to(dev).eval())
    with pytest.raises(PwgbError, match="at least 7 frames"):
        st.push(mels(1, 6, 1)[0])
    st.push(mels(1, 7, 1)[0])
    st.push(mels(1, 1, 2)[0])  # later pushes may be short
    st.reset()
    with pytest.raises(PwgbError, match="at least 7 frames"):
        st.push(mels(1, 3, 1)[0])
    with pytest.raises(PwgbError):
        CausalMelGANStream(models.MelGANGenerator(**dict(small, use_causal_conv=False)).to(dev).eval())
    with pytest.raises(PwgbError):
        CausalMelGANStream(models.MelGANGenerator(**small).to(dev).train())
    with pytest.raises(PwgbError):
        CausalMelGANStream(models.MelGANGenerator(**small).eval())
    with pytest.raises(PwgbError):
        CausalMelGANStream(models.HiFiGANGenerator(use_causal_conv=True, channels=32).to(dev).eval())
