"""Streaming the discrete-symbol HiFi-GAN on the GPU (parallelwavegan_b200.streaming.DiscreteSymbolHiFiGANLookaheadStream):
the stream embed kernel is bit-identical to the whole-utterance embed on the explicit chunk (index dtypes, speakers and
their latch, the end mask, NaN columns), streamed audio followed by the flush is bit-identical to [zeros(delay) |
inference] for every chunk schedule while the output conv stays on one kernel, slots with different speakers are
independent across a reset and a partial flush, graphs replay what eager runs compute, and the unsupported models
raise."""
import json

import pytest
import torch

from helpers import REL_TOL, golden_weights, load_golden, rel_l2
from oracle import synth
from stream_harness import dev, debug_get  # noqa: F401

pytestmark = pytest.mark.gpu

SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
# the 24 kHz recipes' upsampling (hop 480) on few channels
SYN24 = dict(in_channels=32, out_channels=1, channels=64, num_embs=50, num_spk_embs=4, spk_emb_dim=32, kernel_size=7,
             upsample_scales=[12, 10, 2, 2], upsample_kernel_sizes=[24, 20, 4, 4], resblock_kernel_sizes=[3, 7, 11],
             resblock_dilations=[[1, 3, 5]] * 3)
# whole utterances below 4096 output samples keep the output conv on the generic FFMA kernel on both sides
FRAMES = {"dsym_small": 12, "dsym_vctk": 12, "syn24": 8}


def _model(dev, name, weight_norm=True):
    from parallelwavegan_b200 import models

    if name == "syn24":
        m = models.DiscreteSymbolHiFiGANGenerator(**json.loads(json.dumps(SYN24)))
        m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, 1.15))
    else:
        meta, _ = load_golden(name)
        m = models.DiscreteSymbolHiFiGANGenerator(**meta["kwargs"])
        m.load_state_dict(golden_weights(meta))
    if not weight_norm:
        m.remove_weight_norm()
    return m.to(dev).eval()


def _units(m, B, T, seed, spk=None):
    """(B, T, 2) int64 (symbol, speaker) with every frame's speaker id different (only the first counts), or (B, T)
    symbols for a model without speakers"""
    g = torch.Generator().manual_seed(seed)
    sym = torch.randint(0, m.emb.num_embeddings, (B, T), generator=g)
    if m.num_spk_embs <= 0:
        return sym
    s = torch.randint(0, m.num_spk_embs, (B, T), generator=g) if spk is None else torch.as_tensor(spk)[:, None].expand(B, T)
    return torch.stack([sym, s], -1)


def _stream(st, c, schedule, flush=True):
    outs, j, k = [], 0, 0
    while j < c.shape[1]:
        n = min(schedule[k % len(schedule)], c.shape[1] - j)
        outs.append(st.push(c[:, j:j + n]))
        j, k = j + n, k + 1
    if flush:
        outs.append(st.flush())
    return torch.cat(outs, -1)


def _expected(m, c, delay):
    """[zeros(delay) | model.inference] of each item alone"""
    d = next(m.parameters()).device
    with torch.no_grad():
        y = torch.stack([m.inference(c[b].reshape(c.shape[1], -1).to(d)).t() for b in range(c.shape[0])])
    return torch.cat([y.new_zeros(y.shape[:-1] + (delay,)), y], -1)


# ---------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("dtype", [torch.int64, torch.float32])
@pytest.mark.parametrize("spk", [False, True])
def test_embed_stream_bit_identical_to_whole_embed(dev, dtype, spk):
    """each chunk's columns (after 5 history columns) equal ops.symbol_embed of the explicit chunk with the latched
    speaker; frames at or past a slot's end are +0.0; the rest of the buffer is untouched; NaN columns where the whole
    embed has them"""
    from parallelwavegan_b200 import ops

    B, E, G, Cc, P = 4, 37, 5, 200, 5
    g = torch.Generator().manual_seed(11)
    table = torch.randn(E, Cc, generator=g).to(dev)
    spk_t = torch.randn(G, Cc, generator=g).to(dev) if spk else None
    latch = torch.full((B,), 7, dtype=torch.int32, device=dev)
    fresh = torch.ones(B, dtype=torch.int32, device=dev)
    frame = torch.zeros(B, dtype=torch.int32, device=dev)
    end = torch.full((B,), 2 ** 31 - 1, dtype=torch.int32, device=dev)
    first = torch.tensor([1, 4, G + 2, 0])  # slot 2's speaker is outside the table: every column NaN
    cur = first.clone()
    for step, n in enumerate([1, 33, 6, 70]):
        c = torch.stack([torch.randint(0, E, (B, n), generator=g), torch.randint(0, G, (B, n), generator=g)], 1).to(dtype)
        c[:, 1, 0] = torch.tensor([3, 2, 1, 4])  # a later chunk's first speaker id must not count
        if step == 0:
            c[:, 1, 0] = first
        if step == 2:
            c[0, 0, n // 2] = E + 3  # outside the table
            c[3, 0, 1] = -1
            end[1] = frame[1] + 2  # slot 1 ends inside this chunk
        if dtype == torch.float32:
            c[:, 0] += 0.6  # c.long() truncates
            if step == 3:
                c[0, 0, 5] = float("nan")
        if not spk:
            c = c[:, :1]
        y = torch.randn(B, Cc, P + n + 3, generator=g).to(dev)
        y0 = y.clone()
        ops.symbol_embed_stream(c.to(dev), table, spk_t, latch if spk else None, fresh if spk else None, (frame, end), y, P)
        if spk:
            fresh.zero_()
            assert torch.equal(latch.cpu(), torch.where(first < G, first, -2).int())
        cx = c.clone()
        if spk:
            cx[:, 1, 0] = cur.to(dtype)
        ref = ops.symbol_embed(cx.to(dev), table, spk_t)
        past = (frame[:, None].cpu() + torch.arange(n)) >= end[:, None].cpu()
        ref = torch.where(past[:, None, :].to(dev), torch.zeros((), device=dev), ref)
        assert torch.equal(y[:, :, P:P + n].isnan(), ref.isnan())
        assert torch.equal(torch.nan_to_num(y[:, :, P:P + n], 5.0), torch.nan_to_num(ref, 5.0))
        assert torch.equal(y[:, :, :P], y0[:, :, :P]) and torch.equal(y[:, :, P + n:], y0[:, :, P + n:])
        if step == 2:
            assert torch.equal(y[1, :, P + 2:P + n], torch.zeros_like(y[1, :, P + 2:P + n]))
            assert not torch.signbit(y[1, :, P + 2:P + n]).any()
        assert bool(y[2, :, P:P + n].isnan().all()) == spk
        frame += n


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("weight_norm", [True, False])
@pytest.mark.parametrize("name", ["dsym_small", "dsym_vctk", "syn24"])
def test_stream_equals_inference(dev, name, weight_norm, schedule):
    from parallelwavegan_b200.streaming import DiscreteSymbolHiFiGANLookaheadStream

    m = _model(dev, name, weight_norm)
    c = _units(m, 2, FRAMES[name], 71)
    st = DiscreteSymbolHiFiGANLookaheadStream(m, batch=2)
    ref = _expected(m, c, st.delay)
    assert debug_get(3, 6)[0] == 0  # the output conv of the whole utterance took the generic kernel
    y = _stream(st, c, SCHEDULES[schedule])
    assert debug_get(3, 6)[0] == 0  # and so did the stream's
    assert torch.equal(y, ref)


def test_inference_with_g_and_float_indices(dev):
    """inference(c, g) replaces every speaker id by g; the stream pushes the same (T, 2) rows, as float32 too"""
    from parallelwavegan_b200.streaming import DiscreteSymbolHiFiGANLookaheadStream

    meta, gold = load_golden("dsym_vctk")
    m = _model(dev, "dsym_vctk")
    c = gold["c"][0, :, :FRAMES["dsym_vctk"]].t().long()  # (T, 2)
    with torch.no_grad():
        y_g = m.inference(c.to(dev), g=meta["g"]).t()
    cg = c.clone()
    cg[:, 1] = meta["g"]
    st = DiscreteSymbolHiFiGANLookaheadStream(m)
    ref = torch.cat([y_g.new_zeros(1, st.delay), y_g], -1)[None]
    assert torch.equal(_stream(st, cg[None], SCHEDULES["mixed"]), ref)
    assert torch.equal(_stream(st, cg[None].float() + 0.25, SCHEDULES["short"]), ref)
    # the golden's own output, within the suite's tolerance
    full = gold["c"][0].t()
    y = _stream(st, full[None], SCHEDULES["mixed"])
    assert rel_l2(y[0, :, st.delay:].t().cpu(), gold["y_inf"]) < REL_TOL


def test_out_of_range_indices_give_nan_columns(dev):
    from parallelwavegan_b200.streaming import DiscreteSymbolHiFiGANLookaheadStream

    m = _model(dev, "dsym_small")
    c = _units(m, 1, 10, 72)
    c[0, 6] = 99
    st = DiscreteSymbolHiFiGANLookaheadStream(m)
    y = _stream(st, c, SCHEDULES["short"])
    ref = _expected(m, c, st.delay)
    assert torch.equal(y.isnan(), ref.isnan()) and bool(ref.isnan().any())
    assert torch.equal(torch.nan_to_num(y, 3.0), torch.nan_to_num(ref, 3.0))


def test_delay_from_the_module(dev):
    from oracle.ref_dsym_lookahead_stream import DSymLookaheadRef
    from parallelwavegan_b200.streaming import DiscreteSymbolHiFiGANLookaheadStream

    for name, delay in (("dsym_vctk", 3482), ("syn24", 4526), ("dsym_small", 212)):
        st = DiscreteSymbolHiFiGANLookaheadStream(_model(dev, name))
        assert st.delay == delay, name
        cfg = SYN24 if name == "syn24" else load_golden(name)[0]["kwargs"]
        assert st.delay == DSymLookaheadRef({}, cfg).delay


def test_long_utterance_within_rel_l2(dev):
    """40 frames at hop 320: the whole utterance's output conv takes conv1d_fewcout_long_kernel, whose sum order a
    stream cannot reproduce"""
    from parallelwavegan_b200.streaming import DiscreteSymbolHiFiGANLookaheadStream

    m = _model(dev, "dsym_vctk")
    c = _units(m, 2, 40, 73)
    st = DiscreteSymbolHiFiGANLookaheadStream(m, batch=2)
    ref = _expected(m, c, st.delay)
    assert debug_get(3, 6)[0] == 2
    y = _stream(st, c, SCHEDULES["mixed"])
    assert rel_l2(y.cpu(), ref.cpu()) <= 1e-6


def test_batch_slots_speakers_reset_flush_and_graphs(dev):
    """B = 4 slots with different speakers equal four B = 1 streams, graph replay equals eager, a mid-stream reset of
    one slot restarts only that slot (with a new speaker), and flushing slot 0 leaves slot 1 bit-identical to an
    uninterrupted run"""
    from parallelwavegan_b200.streaming import DiscreteSymbolHiFiGANLookaheadStream

    m = _model(dev, "dsym_vctk")
    T = FRAMES["dsym_vctk"]
    c = _units(m, 4, T, 74)
    y4 = _stream(DiscreteSymbolHiFiGANLookaheadStream(m, batch=4), c, SCHEDULES["mixed"])
    for b in range(4):
        assert torch.equal(y4[b:b + 1], _stream(DiscreteSymbolHiFiGANLookaheadStream(m, batch=1), c[b:b + 1], SCHEDULES["mixed"]))
    assert torch.equal(y4, _expected(m, c, y4.shape[-1] - T * 320))
    assert torch.equal(_stream(DiscreteSymbolHiFiGANLookaheadStream(m, batch=4, use_graphs=False), c, SCHEDULES["mixed"]), y4)
    # slot 1 restarts after 5 frames on a new utterance and speaker; the other slots continue
    st = DiscreteSymbolHiFiGANLookaheadStream(m, batch=4)
    first = _stream(st, c[:, :5], [2, 3], flush=False)
    c2 = c.clone()
    c2[1, 5:] = _units(m, 1, T - 5, 75)[0]
    st.reset(1)
    rest = _stream(st, c2[:, 5:], [1, 3, 5])
    y = torch.cat([first, rest], -1)
    for b in (0, 2, 3):
        assert torch.equal(y[b], y4[b])
    assert torch.equal(rest[1:2], _expected(m, c2[1:2, 5:], st.delay))
    # slot 0 ends after 4 frames and is flushed while slot 1 keeps streaming; slot 2 is flushed before its first push
    # and keeps its fresh latch
    st = DiscreteSymbolHiFiGANLookaheadStream(m, batch=3)
    a = st.push(c[:3, :4])
    st.reset(2)
    f0 = st.flush(0)
    assert f0.shape == (1, 1, st.delay)
    assert torch.equal(torch.cat([a[:1], f0], -1), _expected(m, c[:1, :4], st.delay))
    st.flush(2)
    rest = _stream(st, c[:3, 4:], [3, 1, 6])
    uninterrupted = _stream(DiscreteSymbolHiFiGANLookaheadStream(m, batch=1), c[1:2], SCHEDULES["mixed"])
    assert torch.equal(torch.cat([a[1:2], rest[1:2]], -1), uninterrupted)
    assert torch.equal(rest[:1], _expected(m, c[:1, 4:], st.delay))
    assert torch.equal(rest[2:3], _expected(m, c[2:3, 4:], st.delay))


def test_state_bytes(dev):
    from parallelwavegan_b200.streaming import DiscreteSymbolHiFiGANLookaheadStream

    st = DiscreteSymbolHiFiGANLookaheadStream(_model(dev, "dsym_vctk"), batch=3)
    assert st.state_bytes() == sum(t[0].numel() * t.element_size() for t in st._state())


def test_unsupported_models_raise(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import DiscreteSymbolHiFiGANLookaheadStream

    small = dict(in_channels=16, channels=32, num_embs=10, num_spk_embs=0, upsample_scales=[4, 2], upsample_kernel_sizes=[8, 4])
    with pytest.raises(PwgbError, match="train mode"):
        DiscreteSymbolHiFiGANLookaheadStream(models.DiscreteSymbolHiFiGANGenerator(**small).to(dev).train())
    with pytest.raises(PwgbError, match="CUDA"):
        DiscreteSymbolHiFiGANLookaheadStream(models.DiscreteSymbolHiFiGANGenerator(**small).eval())
    with pytest.raises(PwgbError, match="concat_spk_emb"):
        DiscreteSymbolHiFiGANLookaheadStream(models.DiscreteSymbolHiFiGANGenerator(
            **dict(small, num_spk_embs=4, spk_emb_dim=8, concat_spk_emb=True)).to(dev).eval())
    for scales, kernels in (([3, 2], [6, 4]), ([4, 2], [8, 6]), ([4, 2], [12, 4])):
        with pytest.raises(PwgbError, match="kernel 2 \\* stride"):
            DiscreteSymbolHiFiGANLookaheadStream(models.DiscreteSymbolHiFiGANGenerator(
                **dict(small, upsample_scales=scales, upsample_kernel_sizes=kernels)).to(dev).eval())
    for other in (models.DiscreteSymbolDurationGenerator(**dict(small, num_embs=9)), models.HiFiGANGenerator(channels=32)):
        with pytest.raises(PwgbError, match="expected a DiscreteSymbolHiFiGANGenerator"):
            DiscreteSymbolHiFiGANLookaheadStream(other.to(dev).eval())
    st = DiscreteSymbolHiFiGANLookaheadStream(models.DiscreteSymbolHiFiGANGenerator(**dict(small, num_spk_embs=4, spk_emb_dim=16))
                                              .to(dev).eval(), batch=2)
    with pytest.raises(PwgbError, match="push"):
        st.push(torch.zeros(2, 3, dtype=torch.int64))  # speakers missing


# ---------------------------------------------------------------------------------------------------- duration model
DUR_SYN = dict(in_channels=48, out_channels=1, channels=64, num_embs=30, num_spk_embs=0, duration_chans=64, kernel_size=7,
               upsample_scales=[4, 2], upsample_kernel_sizes=[8, 4], resblock_kernel_sizes=[3, 7], resblock_dilations=[[1, 3], [1, 3]])


def _dur_model(dev, name, bias=None):
    from parallelwavegan_b200 import models

    if name == "dur_syn":
        m = models.DiscreteSymbolDurationGenerator(**DUR_SYN)
        m.load_state_dict(synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 41, 1.15))
        with torch.no_grad():
            m.duration_predictor.linear.bias.fill_(1.2)  # durations of 0 .. 6 frames
    else:
        meta, _ = load_golden(name)
        m = models.DiscreteSymbolDurationGenerator(**meta["kwargs"])
        m.load_state_dict(golden_weights(meta))
        with torch.no_grad():
            m.duration_predictor.linear.bias.fill_(meta["linear_bias"])
            m.duration_predictor.linear.weight.mul_(meta["linear_weight_scale"])
    if bias is not None:
        with torch.no_grad():
            m.duration_predictor.linear.bias.fill_(bias)
    return m.to(dev).eval()


def _dur_stream(st, c, schedule):
    """c (B, S) pushed in pushes of ``schedule`` symbols, then flushed -> (per-slot audio list, per-slot durations list)"""
    B = c.shape[0]
    outs, durs, j, k = [[] for _ in range(B)], [[] for _ in range(B)], 0, 0
    while j < c.shape[1]:
        n = min(schedule[k % len(schedule)], c.shape[1] - j)
        y = st.push(c[:, j:j + n])
        for b in range(B):
            outs[b].append(y[b])
            durs[b].append(st.last_durations[b])
        j, k = j + n, k + 1
    fl = st.flush()
    for b in range(B):
        outs[b].append(fl[b])
        durs[b].append(st.last_durations[b])
    return [torch.cat(o, -1) for o in outs], [torch.cat(d) for d in durs]


def _synthesis(m, c_b, delay):
    with torch.no_grad():
        y, ds = m.synthesis(c_b.view(1, 1, -1).to(next(m.parameters()).device))
    return torch.cat([y.new_zeros(1, delay), y[0]], -1), ds[0].cpu()


def test_regulate_kernel_bit_identical_to_whole_regulation(dev):
    """B = 4 queues with zero durations and runs longer than a push, drained in pushes of 1, 4, 2, 7 ... frames whose
    heads differ per slot, equal ops.symbol_embed(..., ds=...) on the whole symbol row"""
    from parallelwavegan_b200 import ops

    B, S, E, Cc = 4, 23, 40, 96
    g = torch.Generator().manual_seed(21)
    table = torch.randn(E, Cc, generator=g).to(dev)
    ids = torch.randint(0, E, (B, S), generator=g)
    ids[1, 3] = E + 2  # outside the table: NaN frames
    ds = torch.randint(0, 4, (B, S), generator=g)
    ds[0, 5], ds[2, 0], ds[3, 7] = 11, 0, 9
    q = ops.DurationQueue(B, 64, dev)
    frame = torch.zeros(B, dtype=torch.int32, device=dev)
    end = torch.full((B,), 2 ** 31 - 1, dtype=torch.int32, device=dev)
    # append with log-durations that round to ds: log(ds + 1)
    x = torch.log(ds.double() + 1.0).float().to(dev)
    ops.duration_queue_append(q, x, ids.to(dev).contiguous(), (frame, end), 0, 1.0)
    frame += S
    assert torch.equal(q.counts[:, 0].cpu(), ds.sum(1))
    ref = ops.symbol_embed(ids.view(B, 1, S).to(dev), table, ds=ds.to(dev), t_out=int(ds.sum(1).max()))
    tot = ds.sum(1)
    outs, j = [], 0
    fz = torch.zeros(B, dtype=torch.int32, device=dev)
    for n in [1, 4, 2, 7, 3, 16] * 4:
        if j >= int(tot.min()):
            break
        n = min(n, int(tot.min()) - j)
        y = torch.randn(B, Cc, n + 3, generator=g).to(dev)
        ops.symbol_regulate_stream(table, q, (fz, end), y, 3, n)
        outs.append(y[:, :, 3:])
        j += n
    y = torch.cat(outs, -1)
    r = ref[:, :, :y.shape[-1]]
    assert torch.equal(y.isnan(), r.isnan()) and torch.equal(torch.nan_to_num(y, 2.0), torch.nan_to_num(r, 2.0))
    assert torch.equal(q.counts[:, 0].cpu(), tot - j)


@pytest.mark.parametrize("schedule", ["ones", "mixed", "long"])
@pytest.mark.parametrize("weight_norm", [True, False])
def test_duration_stream_equals_synthesis_cvss(dev, weight_norm, schedule):
    """the dsym_dur_cvss fixture, both items in one batch: durations equal the fixture's ds_syn and synthesis's, the audio
    equals [zeros(delay) | synthesis] bit for bit (below 4096 samples)"""
    from parallelwavegan_b200.streaming import DiscreteSymbolDurationLookaheadStream

    _, gold = load_golden("dsym_dur_cvss")
    m = _dur_model(dev, "dsym_dur_cvss")
    if not weight_norm:
        m.remove_weight_norm()
    c = gold["c"][:, 0].long()
    st = DiscreteSymbolDurationLookaheadStream(m, batch=2)
    assert st.P == 2
    ys, ds = _dur_stream(st, c, SCHEDULES[schedule])
    for b in range(2):
        ref, dref = _synthesis(m, c[b], st.delay)
        assert torch.equal(ds[b], dref) and torch.equal(ds[b], gold["ds_syn"][b])
        assert torch.equal(ys[b], ref)


def test_duration_stream_synthetic_slots_stalls_and_graphs(dev):
    """an even-stride synthetic model: B = 3 slots with different units (one stalls the others while its durations are
    zero) each equal their own synthesis; graphs equal eager"""
    from parallelwavegan_b200.streaming import DiscreteSymbolDurationLookaheadStream

    m = _dur_model(dev, "dur_syn")
    g = torch.Generator().manual_seed(9)
    c = torch.randint(0, DUR_SYN["num_embs"] + 1, (3, 19), generator=g)
    st = DiscreteSymbolDurationLookaheadStream(m, batch=3)
    ys, ds = _dur_stream(st, c, SCHEDULES["mixed"])
    for b in range(3):
        ref, dref = _synthesis(m, c[b], st.delay)
        assert int(dref.min()) == 0 and int(dref.max()) >= 2
        assert torch.equal(ds[b], dref)
        assert torch.equal(ys[b], ref)
    ys2, _ = _dur_stream(DiscreteSymbolDurationLookaheadStream(m, batch=3, use_graphs=False), c, SCHEDULES["mixed"])
    for b in range(3):
        assert torch.equal(ys2[b], ys[b])


def test_duration_stream_all_zero_predictor(dev):
    """a very negative linear bias: every duration rounds to 0; each slot alone gets unit durations at its flush, and
    equals inference (synthesis of a batch of one)"""
    from parallelwavegan_b200.streaming import DiscreteSymbolDurationLookaheadStream

    m = _dur_model(dev, "dur_syn", bias=-30.0)
    g = torch.Generator().manual_seed(10)
    c = torch.randint(0, DUR_SYN["num_embs"], (2, 9), generator=g)
    st = DiscreteSymbolDurationLookaheadStream(m, batch=2)
    for j in range(0, 9, 3):
        assert st.push(c[:, j:j + 3]).shape[-1] == 0  # nothing is queued before the flush
    fl = st.flush()
    for b in range(2):
        with torch.no_grad():
            y = m.inference(c[b].view(-1, 1).to(dev)).t()
        assert y.shape[-1] == 9 * 8
        assert torch.equal(fl[b], torch.cat([y.new_zeros(1, st.delay), y], -1))


def test_duration_stream_queue_overflow_raises(dev):
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import DiscreteSymbolDurationLookaheadStream

    st = DiscreteSymbolDurationLookaheadStream(_dur_model(dev, "dur_syn", bias=-30.0), max_queue=4)
    with pytest.raises(PwgbError, match="max_queue"):
        st.push(torch.arange(9).view(1, 9))


def test_duration_stream_refusals(dev):
    from parallelwavegan_b200 import models
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import DiscreteSymbolDurationLookaheadStream

    with pytest.raises(PwgbError, match="speakers"):
        DiscreteSymbolDurationLookaheadStream(models.DiscreteSymbolDurationGenerator(
            **dict(DUR_SYN, num_spk_embs=4, spk_emb_dim=48)).to(dev).eval())
    with pytest.raises(PwgbError, match="expected a DiscreteSymbolDurationGenerator"):
        DiscreteSymbolDurationLookaheadStream(models.DiscreteSymbolHiFiGANGenerator(num_spk_embs=0, channels=32).to(dev).eval())
    with pytest.raises(PwgbError, match="train mode"):
        DiscreteSymbolDurationLookaheadStream(models.DiscreteSymbolDurationGenerator(**DUR_SYN).to(dev).train())
    with pytest.raises(PwgbError, match="CUDA"):
        DiscreteSymbolDurationLookaheadStream(models.DiscreteSymbolDurationGenerator(**DUR_SYN).eval())
    with pytest.raises(PwgbError, match="kernel 2 \\* stride"):
        DiscreteSymbolDurationLookaheadStream(models.DiscreteSymbolDurationGenerator(
            **dict(DUR_SYN, upsample_scales=[3, 2], upsample_kernel_sizes=[6, 4])).to(dev).eval())
