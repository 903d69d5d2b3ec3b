"""Streaming the centred (multi-band) MelGAN on the GPU (parallelwavegan_b200.streaming.MelGANLookaheadStream): the
history convs with the reflect / replicate edge policy are bit-identical to the whole-signal conv with that pad on both
engines and every tensor-core plan, streamed audio followed by the flush is bit-identical to [zeros(delay) | inference]
for every chunk schedule and pad, slots are independent (also across a flush), graphs replay what eager runs compute,
and the unsupported models and too-short flushes raise."""
import json

import pytest
import torch

from helpers import REL_TOL, golden_weights, load_golden, rel_l2
from oracle import synth
from stream_harness import dev, debug_get, mels  # noqa: F401

pytestmark = pytest.mark.gpu

# one frame at a time (from a fresh slot), 3 frames, 7 frames and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
PADS = {"reflect": {}, "replicate": dict(pad="ReplicationPad1d"), "zero": dict(pad="ConstantPad1d", pad_params={"value": 0.0})}
V1 = dict(in_channels=80, out_channels=1, kernel_size=7, channels=512, upsample_scales=[8, 8, 2, 2], stack_kernel_size=3, stacks=3)
MB2 = dict(in_channels=80, out_channels=4, kernel_size=7, channels=384, upsample_scales=[8, 4, 2], stack_kernel_size=3, stacks=4)
MB2_CSMSC = dict(MB2, upsample_scales=[5, 5, 3])
# below the length from which the whole utterance's output conv takes conv1d_fewcout_long_kernel (4096 samples)
FRAMES = {"v1": 15, "mb2": 63, "mb2_csmsc": 54}
GOLDEN = ["melgan_small", "melgan_centred_replicate", "melgan_centred_zero", "mb_melgan_v2", "melgan_centred_mb"]


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


def _synthetic(dev, kind, weight_norm=True, pad="reflect"):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.layers import PQMF

    kw = dict({"v1": V1, "mb2": MB2, "mb2_csmsc": MB2_CSMSC}[kind], **PADS[pad])
    m = models.MelGANGenerator(**json.loads(json.dumps(kw)))
    m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 9, 1.0))
    if not weight_norm:
        m.remove_weight_norm()
    m = m.to(dev).eval()
    if kind != "v1":
        m.pqmf = PQMF(4).to(dev)
    return m


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
    """[zeros(delay) | model.inference] of each item alone: (B, 1, delay + T * hop * subbands)"""
    d = next(m.parameters()).device
    with torch.no_grad():
        y = torch.stack([m.inference(c[b].to(d)).t() for b in range(c.shape[0])])
    return torch.cat([y.new_zeros(y.shape[:-1] + (delay,)), y], -1)


# ---------------------------------------------------------------------------------------------------- kernels
# name: cin, cout, K, dilation, n, epilogue, engine, expected tensor-core plan (history (K - 1) d = the conv's pad_left)
ECASES = {
    "tc_cp": (64, 64, 3, 2, 300, "res", "tc", "cp"),
    "tc_direct": (32, 32, 3, 176, 100, "plain", "tc", "direct"),
    "tc_win": (32, 32, 3, 1100, 500, "res", "tc", "win"),
    "tc_nco": (32, 256, 11, 5, 700, "res", "tc", "nco"),
    "ffma_dilated": (16, 8, 3, 3, 257, "res", "simt", None),
    "ffma_out_conv": (48, 4, 7, 1, 90, "plain", "simt", None),
    "ffma_tanh": (32, 1, 7, 1, 1500, "tanh", "simt", None),
}


@pytest.mark.parametrize("pad", ["reflect", "replicate"])
@pytest.mark.parametrize("name", list(ECASES))
def test_conv_stream_edge_bit_exact(dev, name, pad):
    """Three slots in one launch: one at the start of its signal, one mid-signal and one whose signal ends inside the
    window, with the mask, a delayed residual and rows outside the signal holding garbage.  Every output inside the
    signal equals the whole-signal conv with the pad (pwgb_conv1d_forward / pwgb_conv1d_tc_forward), the others +0.0."""
    from parallelwavegan_b200 import ops

    cin, cout, K, d, n, epi, engine, plan = ECASES[name]
    B, H, p, rate = 3, (K - 1) * d, (K - 1) * d // 2, 2
    g = torch.Generator().manual_seed(sum(map(ord, name + pad)))
    look_in = n // 3
    look_out = look_in + p
    f_mid = (look_in + H) // rate + 3
    frames = [0, f_mid, f_mid]
    u = torch.tensor(frames)[:, None] * rate - look_in + torch.arange(-H, n)  # signal sample of each row of [hist | x]
    u_max = int(u[:, -1].max())
    Ls = [u_max + p + 2, u_max + p + 2, int(u[2, H + n // 2]) // rate * rate]
    end = torch.tensor([2 ** 31 - 1, 2 ** 31 - 1, Ls[2] // rate], dtype=torch.int32, device=dev)
    frame = torch.tensor(frames, dtype=torch.int32, device=dev)
    S = [torch.randn(cin, L, generator=g) for L in Ls]
    xp = torch.randn(B, cin, H + n, generator=g)  # garbage outside the signal
    for b in range(B):
        ok = (u[b] >= 0) & (u[b] < Ls[b])
        xp[b][:, ok] = S[b][:, u[b][ok]]
    hist, x = xp[..., :H].contiguous().to(dev), xp[..., H:].contiguous().to(dev)
    w = (torch.randn(cout, cin, K, generator=g) / (cin * K) ** 0.5).to(dev)
    bias = torch.randn(cout, generator=g).to(dev)
    kw = dict(pre_slope=0.2)
    if epi == "tanh":
        kw.update(pre_slope=0.2, post_act="tanh")
    Hr, rd = 9, 5
    r = torch.randn(B, cout, n, generator=g)
    rh = torch.randn(B, cout, Hr, generator=g)
    r_eff = torch.cat([rh, r], -1)[..., Hr - rd:Hr - rd + n]
    old = ops.ENGINE
    ops.ENGINE = "simt" if engine == "simt" else "auto"
    try:
        res = dict(residual=r.to(dev), res_hist=rh.to(dev), res_delay=rd) if epi == "res" else {}
        y = ops.conv1d_stream(x, hist, w, bias, pad_left=H, dilation=d, mask=(frame, end, rate, look_out), edge=pad,
                              in_lookahead=look_in, **res, **kw)
        if engine == "tc":
            pl = debug_get(1, 8)
            assert pl[5] == 0 and {"cp": pl[3] > 0 and not pl[6], "direct": pl[3] == 0, "win": pl[6] == 1, "nco": pl[7] > 1}[plan], pl
        else:
            assert debug_get(3, 6)[0] == 0
        ref = torch.zeros(B, cout, n)
        for b in range(B):
            o = frames[b] * rate - look_out + torch.arange(n)
            inside = (o >= 0) & (o < Ls[b])
            rw = torch.zeros(1, cout, Ls[b])
            rw[0][:, o[inside]] = r_eff[b][:, inside]
            whole = ops.conv1d_raw(S[b][None].to(dev), w, bias, dilation=d, padding=p, pad_mode=pad, **kw,
                                   **(dict(residual=rw.to(dev)) if epi == "res" else {})).cpu()
            ref[b][:, inside] = whole[0][:, o[inside]]
    finally:
        ops.ENGINE = old
    assert torch.equal(y.cpu(), ref)


def test_edge_policy_refusals(dev):
    from parallelwavegan_b200 import ops
    from parallelwavegan_b200.capi import PwgbError

    x = torch.randn(2, 8, 10, device=dev)
    w = torch.randn(8, 8, 3, device=dev)
    frame = torch.zeros(2, dtype=torch.int32, device=dev)
    end = torch.full((2,), 2 ** 31 - 1, dtype=torch.int32, device=dev)
    with pytest.raises(PwgbError, match="mask"):
        ops.conv1d_stream(x, None, w, pad_left=2, edge="reflect")
    with pytest.raises(PwgbError):
        ops.conv1d_stream(x, None, w, pad_left=2, mask=(frame, end, 1, 0), edge="circular")
    with pytest.raises(PwgbError, match="in_lookahead"):
        ops.conv1d_stream(x, None, w, pad_left=2, mask=(frame, end, 1, 0), edge="reflect", in_lookahead=-1)


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("weight_norm", [True, False])
@pytest.mark.parametrize("name", GOLDEN)
def test_golden_stream_equals_inference(dev, name, weight_norm, schedule):
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    meta, _, m = _golden(dev, name, weight_norm)
    c = mels(2, 13, 71)
    st = MelGANLookaheadStream(m, batch=2)
    ref = _expected(m, c, st.delay)
    y = _stream(st, c, SCHEDULES[schedule])
    assert torch.equal(y, ref)


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("pad", list(PADS))
@pytest.mark.parametrize("kind", ["v1", "mb2", "mb2_csmsc"])
def test_stream_equals_inference(dev, kind, pad, schedule):
    """MelGAN v1 (512 channels) and multi-band MelGAN v2 at both recipes' scales, all three pads"""
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    m = _synthetic(dev, kind, pad=pad)
    c = mels(1, FRAMES[kind], 72)
    st = MelGANLookaheadStream(m)
    ref = _expected(m, c, st.delay)
    if kind == "v1":
        assert debug_get(3, 6)[0] == 0  # the output conv of the whole utterance took the generic kernel
    assert torch.equal(_stream(st, c, SCHEDULES[schedule]), ref)


@pytest.mark.parametrize("kind", ["v1", "mb2"])
def test_stream_without_weight_norm(dev, kind):
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    m = _synthetic(dev, kind, weight_norm=False)
    c = mels(2, 11, 73)
    st = MelGANLookaheadStream(m, batch=2)
    assert torch.equal(_stream(st, c, SCHEDULES["mixed"]), _expected(m, c, st.delay))


@pytest.mark.parametrize("pad", list(PADS))
@pytest.mark.parametrize("kind", ["v1", "mb2", "mb2_csmsc"])
def test_shortest_utterances_come_from_the_flush(dev, kind, pad):
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    m = _synthetic(dev, kind, pad=pad)
    st = MelGANLookaheadStream(m, batch=2)
    assert st.min_frames == ({"v1": 4, "mb2": 4, "mb2_csmsc": 6}[kind] if pad == "reflect" else 1)
    c = mels(2, st.min_frames, 74)
    for schedule in (SCHEDULES["ones"], SCHEDULES["long"]):
        assert torch.equal(_stream(st, c, schedule), _expected(m, c, st.delay))


def test_delays_from_the_module(dev):
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    assert MelGANLookaheadStream(_synthetic(dev, "v1")).delay == 1425
    assert MelGANLookaheadStream(_synthetic(dev, "mb2")).delay == 4 * 672 + 31
    assert MelGANLookaheadStream(_synthetic(dev, "mb2_csmsc")).delay == 4 * 1044 + 31


@pytest.mark.parametrize("name", GOLDEN)
def test_stream_matches_reference_output(dev, name):
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    meta, g, m = _golden(dev, name)
    c = synth.randn(meta["c_shape"], meta["c_seed"])[0].t()
    st = MelGANLookaheadStream(m)
    y = _stream(st, c[None], SCHEDULES["mixed"])
    assert rel_l2(y[0, :, st.delay:].t().cpu(), g["y_inf"] if "y_inf" in g else g["y"][0].t()) < REL_TOL


def test_long_utterance_within_rel_l2(dev):
    """48 frames of v1: the whole utterance's output conv takes conv1d_fewcout_long_kernel, whose sum order a stream
    cannot reproduce"""
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    m = _synthetic(dev, "v1")
    c = mels(1, 48, 75)
    st = MelGANLookaheadStream(m)
    ref = _expected(m, c, st.delay)
    assert debug_get(3, 6)[0] == 2
    assert rel_l2(_stream(st, c, SCHEDULES["mixed"]).cpu(), ref.cpu()) <= 1e-6


def test_batch_slots_reset_flush_and_graphs(dev):
    """B = 4 equals four B = 1 streams, graph replay equals eager, a mid-stream reset of one slot restarts only that
    slot, and flushing slot 0 leaves slot 1's whole output bit-identical to an uninterrupted run"""
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    m = _synthetic(dev, "mb2")
    T = 30
    c = mels(4, T, 76)
    y4 = _stream(MelGANLookaheadStream(m, batch=4), c, SCHEDULES["mixed"])
    for b in range(4):
        assert torch.equal(y4[b:b + 1], _stream(MelGANLookaheadStream(m, batch=1), c[b:b + 1], SCHEDULES["mixed"]))
    assert torch.equal(_stream(MelGANLookaheadStream(m, batch=4, use_graphs=False), c, SCHEDULES["mixed"]), y4)
    # slot 1 restarts after 6 frames on a new utterance; the other slots continue
    st = MelGANLookaheadStream(m, batch=4)
    first = _stream(st, c[:, :6], [2, 4], flush=False)
    c2 = c.clone()
    c2[1, 6:] = mels(1, T - 6, 77)[0]
    st.reset(1)
    rest = _stream(st, c2[:, 6:], [1, 3, 5])
    y = torch.cat([first, rest], -1)
    for b in (0, 2, 3):
        assert torch.equal(y[b], y4[b])
    assert torch.equal(rest[1:2], _expected(m, c2[1:2, 6:], st.delay))
    # slot 0 ends after 5 frames and is flushed while slot 1 keeps streaming
    st = MelGANLookaheadStream(m, batch=2)
    a = st.push(c[:2, :5])
    f0 = st.flush(0)
    assert f0.shape == (1, 1, st.delay)
    assert torch.equal(torch.cat([a[:1], f0], -1), _expected(m, c[:1, :5], st.delay))
    rest = _stream(st, c[:2, 5:], [3, 1, 6])
    uninterrupted = _stream(MelGANLookaheadStream(m, batch=1), c[1:2], SCHEDULES["mixed"])
    assert torch.equal(torch.cat([a[1:2], rest[1:2]], -1), uninterrupted)
    assert torch.equal(rest[:1], _expected(m, c[:1, 5:], st.delay))


def test_more_chunk_lengths_than_cached(dev):
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    _, _, m = _golden(dev, "melgan_centred_mb")
    st = MelGANLookaheadStream(m, batch=2)
    sched = list(range(1, st.MAX_CHUNK_LENGTHS + 3))
    c = mels(2, sum(sched), 78)
    assert torch.equal(_stream(st, c, sched), _expected(m, c, st.delay))


def test_state_bytes(dev):
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    st = MelGANLookaheadStream(_golden(dev, "melgan_centred_mb")[2], batch=3)
    assert st.state_bytes() == sum(t[0].numel() * t.element_size() for t in st._state())
    assert st.state_bytes() == sum(t[0].numel() * t.element_size() for t in st._histories()) + 8


def test_short_flush_raises_and_leaves_state(dev):
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    m = _synthetic(dev, "mb2_csmsc")
    st = MelGANLookaheadStream(m, batch=2)
    c = mels(2, 9, 79)
    a = st.push(c[:, :5])
    snap = [t.clone() for t in st._state()]
    with pytest.raises(PwgbError, match="fewer than 6 frames"):
        st.flush()
    assert all(torch.equal(t, s) for t, s in zip(st._state(), snap))
    rest = _stream(st, c[:, 5:], [4])
    assert torch.equal(torch.cat([a, rest], -1), _expected(m, c, st.delay))


def test_unsupported_models_raise(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.layers import PQMF
    from parallelwavegan_b200.streaming import MelGANLookaheadStream

    small = dict(V1, channels=256)
    with pytest.raises(PwgbError, match="CausalMelGANStream"):
        MelGANLookaheadStream(models.MelGANGenerator(**dict(small, use_causal_conv=True)).to(dev).eval())
    with pytest.raises(PwgbError, match="train mode"):
        MelGANLookaheadStream(models.MelGANGenerator(**small).to(dev).train())
    with pytest.raises(PwgbError, match="CUDA"):
        MelGANLookaheadStream(models.MelGANGenerator(**small).eval())
    m = models.MelGANGenerator(**small).to(dev).eval()
    m.pqmf = PQMF(4).to(dev)
    with pytest.raises(PwgbError, match="PQMF"):
        MelGANLookaheadStream(m)
    for other in (models.HiFiGANGenerator(), models.ParallelWaveGANGenerator()):
        with pytest.raises(PwgbError, match="expected a MelGANGenerator"):
            MelGANLookaheadStream(other.to(dev).eval())
