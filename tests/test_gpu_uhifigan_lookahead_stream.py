"""UHiFiGANLookaheadStream on the GPU.  Its three stream entry points, each bit for bit against the whole-signal call it
stands for: the space-to-depth gather with its history (pwgb_s2d_stream_forward) and the stride-1 conv after it against
``conv1d`` with stride on the whole signal, the FFMA strided history conv (pwgb_conv1d_strided_stream_ext_forward)
against pwgb_conv1d_forward with stride, and the two-source stream conv-transpose
(pwgb_conv_transpose1d_cat_stream_ext_forward) against pwgb_conv_transpose1d_cat_forward on the explicit windows.  The
pushes and the flush of a centred U-Net HiFi-GAN equal [zeros(delay) |
model.inference(excitation, c)] bit for bit for the three golden models, with and without weight norm, on both conv
engines and for several chunk schedules, while the whole-utterance output conv (32 -> 1) has fewer than 4096 samples;
from 4096 on it takes conv1d_fewcout_long_kernel, which sums in another order than the stream's output conv, and the
check is rel-L2 <= 1e-6.  Slots, reset, partial flush, graphs, state size and refusals."""
import pytest
import torch

from helpers import golden_weights, load_golden
from oracle import synth
from stream_harness import dev  # noqa: F401

pytestmark = pytest.mark.gpu

SCHEDULES = {"ones": [1], "short": [3], "mixed": [1, 4, 2, 9, 1, 3]}
LONG_OUTPUT_CONV = 4096  # whole-utterance output samples from which the output conv sums in another order
GOLDENS = ["uhifigan_small", "uhifigan_odd", "uhifigan_opencpop"]


@pytest.fixture
def engine():
    from parallelwavegan_b200 import ops

    saved = ops.ENGINE
    yield ops
    ops.ENGINE = saved


def _model(dev, name, weight_norm=True):
    from parallelwavegan_b200 import models

    meta, _ = load_golden(name)
    m = models.UHiFiGANGenerator(**meta["kwargs"])
    m.load_state_dict(golden_weights(meta))
    if not weight_norm:
        m.remove_weight_norm()
    return m.to(dev).eval(), meta


def _inputs(meta, B=1, frames=None, seed=0):
    T = frames or meta["c_shape"][-1]
    c = synth.randn((B, T, 80), meta["c_seed"] + seed)
    e = synth.randn((B, T * meta["hop"]), meta["e_seed"] + seed, meta["e_scale"])
    return c, e


def _expected(m, c, e, delay):
    """[zeros(delay) | inference] per slot: (B, out_channels, delay + T * hop)"""
    outs, dev = [], next(m.parameters()).device
    with torch.no_grad():
        for b in range(c.shape[0]):
            y = m.inference(excitation=e[b].to(dev), c=c[b].to(dev))
            outs.append(torch.cat([y.new_zeros(delay, y.shape[1]), y]).t())
    return torch.stack(outs)


def _stream(st, c, e, schedule):
    hop = st.hop
    outs, j, k = [], 0, 0
    while j < c.shape[1]:
        n = min(schedule[k % len(schedule)], c.shape[1] - j)
        outs.append(st.push(c[:, j:j + n], e[:, j * hop:(j + n) * hop]))
        j, k = j + n, k + 1
    outs.append(st.flush())
    return torch.cat(outs, -1)


@pytest.mark.parametrize("simt", [False, True])
@pytest.mark.parametrize("weight_norm", [True, False])
@pytest.mark.parametrize("name", GOLDENS)
def test_stream_equals_inference_bit_for_bit(dev, engine, name, weight_norm, simt):
    if simt:
        engine.ENGINE = "simt"
    from parallelwavegan_b200.streaming import UHiFiGANLookaheadStream

    m, meta = _model(dev, name, weight_norm)
    c, e = _inputs(meta)
    hop = meta["hop"]
    short = (LONG_OUTPUT_CONV - 1) // hop  # the longest utterance whose inference is bit-identical
    for use_graphs in (False, True):
        st = UHiFiGANLookaheadStream(m, use_graphs=use_graphs)
        for frames in sorted({min(short, c.shape[1]), c.shape[1]}):
            cf, ef = c[:, :frames], e[:, :frames * hop]
            ref = _expected(m, cf, ef, st.delay)
            for sched in SCHEDULES.values():
                y = _stream(st, cf, ef, sched)
                assert y.shape == ref.shape
                if frames * hop < LONG_OUTPUT_CONV:
                    assert torch.equal(y, ref), (name, frames, sched, float((y - ref).abs().max()))
                else:
                    assert float((y - ref).norm() / ref.norm()) <= 1e-6, (name, frames, sched)


def test_delay_of_the_recipes(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.streaming import UHiFiGANLookaheadStream

    m, _ = _model(dev, "uhifigan_opencpop")
    assert UHiFiGANLookaheadStream(m).delay == 16231
    yesno = models.UHiFiGANGenerator(channels=32, downsample_scales=[2, 2, 8, 8], downsample_kernel_sizes=[4, 4, 16, 16],
                                     dropout=0.1).to(dev).eval()
    assert UHiFiGANLookaheadStream(yesno).delay == 5050


def test_slots_reset_and_partial_flush(dev):
    """B = 4 slots: slot 1 is flushed after 5 frames and starts a new utterance, slot 2 is reset after 3 frames and
    restarts; each slot's audio equals its own utterance's inference, and the flush leaves the others untouched"""
    from parallelwavegan_b200.streaming import UHiFiGANLookaheadStream

    m, meta = _model(dev, "uhifigan_small")
    hop, B, T = meta["hop"], 4, 12
    c, e = _inputs(meta, B, T, seed=7)
    c2, e2 = _inputs(meta, B, T, seed=9)
    st = UHiFiGANLookaheadStream(m, batch=B)
    ref = _expected(m, c, e, st.delay)
    outs = [[] for _ in range(B)]
    tail = None
    for j in range(T):
        # slot 1 runs utterance c2 from frame 5 on, slot 2 restarts c2 at frame 3
        cj = c[:, j:j + 1].clone()
        ej = e[:, j * hop:(j + 1) * hop].clone()
        if j >= 5:
            cj[1], ej[1] = c2[1, j - 5:j - 4], e2[1, (j - 5) * hop:(j - 4) * hop]
        if j >= 3:
            cj[2], ej[2] = c2[2, j - 3:j - 2], e2[2, (j - 3) * hop:(j - 2) * hop]
        if j == 3:
            st.reset(2)
        if j == 5:
            before = [h.clone() for h in st._state()]
            tail = st.flush(1)
            after = st._state()
            for b in (0, 2, 3):
                assert all(torch.equal(x[b], y[b]) for x, y in zip(before, after))
        y = st.push(cj, ej)
        for b in range(B):
            outs[b].append(y[b])
    end = st.flush()
    y0 = torch.cat(outs[0] + [end[0]], -1)
    assert torch.equal(y0, ref[0])
    y3 = torch.cat(outs[3] + [end[3]], -1)
    assert torch.equal(y3, ref[3])
    first1 = torch.cat(outs[1][:5] + [tail[0]], -1)
    assert torch.equal(first1, _expected(m, c[1:2, :5], e[1:2, :5 * hop], st.delay)[0])
    second1 = torch.cat(outs[1][5:] + [end[1]], -1)
    assert torch.equal(second1, _expected(m, c2[1:2, :T - 5], e2[1:2, :(T - 5) * hop], st.delay)[0])
    second2 = torch.cat(outs[2][3:] + [end[2]], -1)
    assert torch.equal(second2, _expected(m, c2[2:3, :T - 3], e2[2:3, :(T - 3) * hop], st.delay)[0])


def test_graphs_match_eager_and_state_bytes(dev):
    from parallelwavegan_b200.streaming import UHiFiGANLookaheadStream

    m, meta = _model(dev, "uhifigan_opencpop")
    c, e = _inputs(meta, 2, 6, seed=3)
    a, b = UHiFiGANLookaheadStream(m, batch=2, use_graphs=False), UHiFiGANLookaheadStream(m, batch=2, use_graphs=True)
    assert torch.equal(_stream(a, c, e, [2, 1]), _stream(b, c, e, [2, 1]))
    # per slot, counted from the float64 oracle's carried tensors (the same plan, restated independently): the
    # excitation, mel and output conv histories, per level the MRF histories, the strided conv's input history and the
    # decoder's two delay lines; plus the two int32 frame counters
    from oracle import ref_uhifigan_lookahead_stream as RU

    ref = RU.UHiFiGANLookaheadRef({}, meta["kwargs"])
    ts = [ref.ein, ref.cin, ref.out]
    for lv in ref.enc + ref.dec:
        mrf = lv["mrf"]
        ts += [mrf.lvl] + [h for hs in mrf.xh + mrf.xth for h in hs]
        ts += [lv["hist"]] if "hist" in lv else [lv["h1"], lv["h2"]]
    assert a.state_bytes() == 4 * sum(t[0].numel() for t in ts) + 8 == 2246176


def test_refusals(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import UHiFiGANLookaheadStream

    m, meta = _model(dev, "uhifigan_small")
    with pytest.raises(PwgbError, match="expected a UHiFiGANGenerator"):
        UHiFiGANLookaheadStream(models.HiFiGANGenerator(channels=32).to(dev).eval())
    with pytest.raises(PwgbError, match="train mode"):
        UHiFiGANLookaheadStream(m.train())
    m.eval()
    with pytest.raises(PwgbError, match="CUDA device"):
        UHiFiGANLookaheadStream(models.UHiFiGANGenerator(**meta["kwargs"]).eval())
    kw = dict(meta["kwargs"], downsample_scales=[2, 2, 2], downsample_kernel_sizes=[4, 4, 4])
    with pytest.raises(PwgbError, match="prod"):
        UHiFiGANLookaheadStream(models.UHiFiGANGenerator(**kw).to(dev).eval())
    kw = dict(meta["kwargs"], downsample_kernel_sizes=[4, 4, 4, 5])
    with pytest.raises(PwgbError, match="kernel 2 \\* stride"):
        UHiFiGANLookaheadStream(models.UHiFiGANGenerator(**kw).to(dev).eval())
    kw = dict(meta["kwargs"], upsample_kernel_sizes=[4, 4, 4, 6])
    with pytest.raises(PwgbError, match="kernel 2 \\* stride"):
        UHiFiGANLookaheadStream(models.UHiFiGANGenerator(**kw).to(dev).eval())
    st = UHiFiGANLookaheadStream(m, batch=2)
    hop = st.hop
    snap = [t.clone() for t in st._state()]
    for c, e in (((2, 3, 79), (2, 3 * hop)), ((2, 3, 80), (2, 3 * hop + 1)), ((2, 3, 80), (2, 2, hop)), ((1, 3, 80), (1, 3 * hop)),
                 ((2, 3, 80), (3 * hop,))):
        with pytest.raises(PwgbError):
            st.push(torch.zeros(c), torch.zeros(e))
    assert all(torch.equal(a, b) for a, b in zip(snap, st._state()))
    # the accepted excitation layouts give the same audio
    c, e = _inputs(meta, 2, 2, seed=5)
    y1 = st.push(c, e)
    st.reset()
    y2 = st.push(c, e.reshape(2, 2, hop))
    assert torch.equal(y1, y2)


# (channels, stride) of the encoder's strided convs: the opencpop recipe's four, then the odd golden config's two
ENCODER_SHAPES = [(32, 5), (64, 5), (128, 4), (256, 3), (32, 3), (64, 5)]


def _strided_case(dev, C, s, seed):
    """x (2, C, T), w (2C, C, 2s), bias, padding p, and an output window [o0, o0 + t) with its padded-input window split
    into a history of H rows (s <= H < 2s, as a stream keeps) and the rows after it"""
    g = torch.Generator().manual_seed(seed)
    T, p = 40 * s, s // 2 + s % 2
    x = torch.randn(2, C, T, generator=g).to(dev)
    w = (torch.randn(2 * C, C, 2 * s, generator=g) * 0.05).to(dev)
    b = (torch.randn(2 * C, generator=g) * 0.1).to(dev)
    cases = []
    for o0, t, H in ((0, 9, s), (7, 13, 2 * s - 1), (30, 10, s + 1)):
        xp = torch.nn.functional.pad(x, (p, 4 * s))  # the whole conv's zero padding, and zeros past the end
        win = xp[:, :, o0 * s:(o0 + t + 1) * s]
        cases.append((o0, t, win[:, :, :H].contiguous(), win[:, :, H:].contiguous()))
    return x, w, b, p, cases


@pytest.mark.parametrize("C, s", ENCODER_SHAPES)
def test_s2d_stream_then_conv_equals_strided_conv(dev, C, s):
    from parallelwavegan_b200 import ops

    x, w, b, p, cases = _strided_case(dev, C, s, 5 + C + s)
    with torch.no_grad():
        whole = ops.conv1d(x, w, b, stride=s, padding=p, post_act="lrelu", post_slope=0.1)
        cgo = (C * s + 31) // 32 * 32
        w2 = ops.s2d_weight(w, s, cgo).contiguous()
        for o0, t, hist, chunk in cases:
            xs = ops.s2d_stream(chunk, hist, s, t + 1, cgo)
            assert torch.equal(xs, ops.s2d_raw(torch.cat([hist, chunk], -1), 1, s, 0, t + 1, 1, cgo))
            y = ops.conv1d_stream(xs, None, w2, b, pad_left=0, post_act="lrelu", post_slope=0.1)
            assert torch.equal(y, whole[:, :, o0:o0 + t]), (C, s, o0)


@pytest.mark.parametrize("C, s", ENCODER_SHAPES)
def test_strided_ffma_stream_conv_equals_strided_conv(dev, engine, C, s):
    engine.ENGINE = "simt"
    ops = engine
    x, w, b, p, cases = _strided_case(dev, C, s, 9 + C + s)
    with torch.no_grad():
        whole = ops.conv1d(x, w, b, stride=s, padding=p, post_act="lrelu", post_slope=0.1)
        for o0, t, hist, chunk in cases:
            y = ops.conv1d_strided_stream(chunk, hist, w, b, stride=s, pad_left=hist.shape[-1], t_out=t, post_act="lrelu",
                                          post_slope=0.1)
            assert torch.equal(y, whole[:, :, o0:o0 + t]), (C, s, o0)


@pytest.mark.parametrize("simt", [False, True])
@pytest.mark.parametrize("delay2", [0, 1, 37])
@pytest.mark.parametrize("C1, C2, cout, s", [(64, 64, 32, 3), (128, 128, 64, 5), (48, 24, 16, 2)])
def test_cat_stream_conv_transpose_equals_cat_forward(dev, engine, C1, C2, cout, s, delay2, simt):
    """the explicit windows: source 1 is [hist1 | x1]; source 2 is rows [-(delay2 + 1), n - delay2) of [hist2 | x2]
    (64 + 64 and 128 + 128 channels take the two-source tensor-core conv-transpose, 48 + 24 the FFMA one on the
    concatenation)"""
    if simt:
        engine.ENGINE = "simt"
    ops = engine
    g = torch.Generator().manual_seed(C1 + C2 + s + delay2)
    B, n, H2 = 2, 6, delay2 + 3
    x1, hist1 = torch.randn(B, C1, n, generator=g).to(dev), torch.randn(B, C1, 1, generator=g).to(dev)
    x2, hist2 = torch.randn(B, C2, n, generator=g).to(dev), torch.randn(B, C2, H2, generator=g).to(dev)
    w = (torch.randn(C1 + C2, cout, 2 * s, generator=g) * 0.05).to(dev)
    b = (torch.randn(cout, generator=g) * 0.1).to(dev)
    with torch.no_grad():
        x1w = torch.cat([hist1, x1], -1)
        x2w = torch.cat([hist2, x2], -1)[:, :, H2 - delay2 - 1:H2 - delay2 + n].contiguous()
        ref = ops.conv_transpose1d_cat_raw(x1w, x2w, w, b, stride=s, padding=s, pre_slope=0.1)
        y = ops.conv_transpose1d_cat_stream(x1, hist1, x2, hist2, delay2, w, b, stride=s, pre_slope=0.1)
    assert y.shape == ref.shape
    assert torch.equal(y, ref)
