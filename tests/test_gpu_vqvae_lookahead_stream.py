"""Streaming a VQ-VAE's wav2wav conversion on the GPU (parallelwavegan_b200.streaming.VQVAELookaheadStream): the grouped
stream entry points are bit-identical to the whole-signal calls on the explicit windows at the encoders' own grouped
shapes, the VQ stream to pwgb_vq_forward with its NaN rules, every encoder layer takes the route ``encode`` takes, the
pushes and flush equal [zeros(delay) | decode(encode(x), l, g)] bit for bit (indices included) for every schedule, with
and without weight norm, for four slots converting to different speakers, across a reset and a partial flush, with
graphs and without; longer signals keep their codes; the unsupported models and inputs raise before any launch."""
import copy
import ctypes as C

import pytest
import torch

from helpers import load_golden, rel_l2
from oracle import synth
from test_vqvae_cpu import vq_weights
from stream_harness import dev, debug_get  # noqa: F401

pytestmark = pytest.mark.gpu
NAMES = ["vqvae_yesno", "vqvae_vctk_g", "vqvae_vctk_lg"]
SCHEDULES = {"ones": [1], "short": [3], "long": [17], "mixed": [1, 4, 2, 9, 1, 3]}


def _model(dev, name, weight_norm=True):
    from parallelwavegan_b200 import models

    meta, g = load_golden(name)
    m = models.VQVAE(**copy.deepcopy(meta["kwargs"]))
    m.load_state_dict(vq_weights(meta, fold=False))
    if not weight_norm:
        m.remove_weight_norm()
    return meta, g, m.to(dev).eval()


def _reference(m, x, l, g):
    with torch.no_grad():
        idx = m.encode(x)
        return idx, m.decode(idx, l, g)


def _stream(st, x, l, g, schedule):
    """pushes of ``schedule`` frames then the flush: (cat(outputs), cat(indices) without the frames outside the signal)"""
    hop, T = st.hop, x.shape[-1] // st.hop
    outs, idx, j, k = [], [], 0, 0
    while j < T:
        n = min(schedule[k % len(schedule)], T - j)
        y, i = st.push(x[..., j * hop:(j + n) * hop], l[..., j:j + n] if l is not None else None, g, return_indices=True)
        outs.append(y)
        idx.append(i)
        j, k = j + n, k + 1
    outs.append(st.flush())
    idx.append(st._entries[-(-st.delay // hop)]["idx"].clone())
    idx = torch.cat(idx, -1)
    return torch.cat(outs, -1), torch.stack([r[r >= 0] for r in idx])


def _check(m, st, x, l, g, schedule):
    ref_idx, ref = _reference(m, x, l, g)
    y, idx = _stream(st, x, l, g, schedule)
    want = torch.cat([torch.zeros(x.shape[0], 1, st.delay, device=x.device), ref], -1)
    assert tuple(y.shape) == tuple(want.shape)
    assert torch.equal(idx, ref_idx)
    assert torch.equal(y, want), float((y - want).abs().max())


# ---------------------------------------------------------------------------------------------------- entry points
# (cin, cout, groups, stride): the strided convs of the yesno and vctk encoders
STRIDED = [(16, 32, 4, 4), (32, 32, 8, 4), (32, 32, 8, 2), (16, 64, 4, 4), (64, 256, 16, 4), (256, 512, 64, 2), (512, 1024, 128, 2)]


@pytest.mark.parametrize("cin,cout,groups,s", STRIDED)
@pytest.mark.parametrize("n", [1, 3, 17])
def test_grouped_strided_entry_points(dev, cin, cout, groups, s, n):
    """each grouped strided launch on [hist | chunk] equals the whole-signal call on the explicit window: the FFMA strided
    stream conv, the grouped space-to-depth and the grouped masked tensor-core conv after it; slots with and without the
    mask's edge inside the chunk"""
    from parallelwavegan_b200 import ops

    K, p = 10 * s + 1, 5 * s
    B, rate = 3, 4
    t_out, H = n * rate, 7 * s + p - 3  # L' = 7 over an input lookahead of 3
    x = synth.randn((B, cin, t_out * s), 100 + n).to(dev)
    hist = synth.randn((B, cin, H), 200 + n).to(dev)
    w = (synth.randn((cout, cin // groups, K), 300) * 0.1).to(dev)
    b = synth.randn((cout,), 301).to(dev)
    win = torch.cat([hist, x], -1)
    frame = torch.tensor([0, 5, 40], device=dev, dtype=torch.int32)
    end = torch.tensor([2 ** 31 - 1, 6, 2 ** 31 - 1], device=dev, dtype=torch.int32)
    mask = (frame, end, rate, 7)

    def masked(y):
        pos = frame[:, None].long() * rate - 7 + torch.arange(y.shape[-1], device=dev)[None]
        keep = (pos >= 0) & (pos < end[:, None].long() * rate)
        return torch.where(keep[:, None], y, torch.zeros((), device=dev))

    want = masked(ops.conv1d_raw(win, w, b, stride=s, groups=groups, post_act="lrelu", post_slope=0.2)[..., :t_out])
    got = ops.conv1d_strided_stream(x, hist, w, b, stride=s, pad_left=H, post_act="lrelu", post_slope=0.2, t_out=t_out, mask=mask,
                                    groups=groups)
    assert torch.equal(got, want)
    cin_g = cin // groups
    cgo = (cin_g * s + 31) // 32 * 32
    rows = t_out + -(-K // s) - 1
    xs = ops.s2d_stream(x, hist, s, rows, cgo, groups=groups)
    assert torch.equal(xs, ops.s2d_raw(win, groups, s, 0, rows, cgo=cgo))
    if (cout // groups) % 16 == 0 and cgo <= 2 * cin_g * s:
        w2 = ops.s2d_weight(w, s, cgo).contiguous()
        ref = ops.conv1d_raw(xs, w2, b, groups=groups, post_act="lrelu", post_slope=0.2)
        plan_whole = debug_get(1, 8)
        got = ops.conv1d_stream(xs, None, w2, b, pad_left=0, post_act="lrelu", post_slope=0.2, mask=mask, groups=groups)
        plan_stream = debug_get(1, 8)
        assert plan_whole[0] == plan_stream[0] and plan_whole[7] == plan_stream[7] == groups * ((cout // groups) // min(cout // groups, 128))
        assert torch.equal(got, masked(ref))


def test_grouped_history_refusals(dev):
    """a grouped tensor-core history launch reads no history: pad_left > 0 is not offered to the tensor cores"""
    from parallelwavegan_b200 import capi

    d = capi.Conv1dDesc(batch=1, cin=128, cout=64, t_in=40, t_out=40, kernel=3, stride=1, dilation=1, groups=4, pad_left=2,
                        pad_mode=capi.PAD_HISTORY, period=1, t_valid=40, pre_slope=1.0, out_scale=1.0)
    assert capi.lib().pwgb_conv1d_tc_supported(C.byref(d)) == 0
    d.pad_left, d.t_out = 0, 38
    assert capi.lib().pwgb_conv1d_tc_supported(C.byref(d)) == 1


@pytest.mark.parametrize("E", [0, 5])
def test_vq_stream_against_vq_forward(dev, E):
    from parallelwavegan_b200 import ops

    torch.manual_seed(7)
    B, D, n, K, Cl, Cg, ng = 4, 64, 21, 40, 8, 16, 6
    z = torch.randn(B, D, n, device=dev)
    z[1, 3, 4] = float("nan")
    cb = torch.randn(K, D, device=dev) * 0.7
    l_hist, l = torch.randn(B, Cl, E, device=dev), torch.randn(B, Cl, n, device=dev)
    gt = torch.randn(ng, Cg, device=dev)
    g = torch.tensor([2, 5, 6, 0], device=dev)  # slot 2: outside the table (NaN columns)
    frame = torch.tensor([0, 9, 30, 100], device=dev, dtype=torch.int32)
    end = torch.tensor([2 ** 31 - 1, 2 ** 31 - 1, 35, 2 ** 31 - 1], device=dev, dtype=torch.int32)
    idx, dec = ops.vq_stream(z, cb, (frame, end, 1, 12), l=l, l_hist=l_hist, global_table=gt, g=g)
    lw = torch.cat([l_hist, l], -1)[..., :n]
    ridx, _, rdec = ops.vq_raw(z, cb, z_q=False, l=lw.contiguous(), global_table=gt, g=g)
    pos = frame[:, None].long() - 12 + torch.arange(n, device=dev)[None]
    keep = (pos >= 0) & (pos < end[:, None].long())
    assert torch.equal(idx, torch.where(keep, ridx, torch.full_like(ridx, -1)))
    want = torch.where(keep[:, None], rdec, torch.zeros((), device=dev))
    assert torch.equal(want.isnan(), dec.isnan()) and torch.equal(torch.nan_to_num(want), torch.nan_to_num(dec))
    assert bool(dec[2][:, keep[2]].isnan().all()) and bool((dec[2][:, ~keep[2]] == 0).all())
    assert int(idx[1, 4]) == 0  # the NaN frame: torch.min's first NaN


def _routes(fn):
    """the conv routes ``fn`` launches, in order: ("tc", MT) or ("ffma", kernel, RCO, WARPS_CO)"""
    from parallelwavegan_b200 import capi

    L = capi.lib()
    names = {"pwgb_conv1d_tc_forward": 1, "pwgb_conv1d_tc_stream_ext_forward": 1, "pwgb_conv1d_forward": 3,
             "pwgb_conv1d_stream_ext_forward": 3, "pwgb_conv1d_strided_stream_ext_forward": 3}
    out, saved = [], {k: getattr(L, k) for k in names}

    def wrap(k, f):
        def call(*a):
            rc = f(*a)
            r = debug_get(names[k], 8 if names[k] == 1 else 6)
            out.append(("tc", r[0]) if names[k] == 1 else ("ffma", r[0], r[1], r[2]))
            return rc
        return call

    try:
        for k, f in saved.items():
            setattr(L, k, wrap(k, f))
        fn()
    finally:
        for k, f in saved.items():
            setattr(L, k, f)
    return out


@pytest.mark.parametrize("name", ["vqvae_yesno", "vqvae_vctk_g"])
def test_encoder_routes_match_encode(dev, name):
    """every encoder layer of the stream takes the engine and kernel family ``encode`` takes at that layer's shape"""
    from parallelwavegan_b200.streaming import VQVAELookaheadStream

    meta, g, m = _model(dev, name)
    x = g["x"].to(dev)
    with torch.no_grad():
        whole = _routes(lambda: m.encoder(x))
    st = VQVAELookaheadStream(m, batch=x.shape[0], use_graphs=False)
    gid = g["g"].to(dev) if "g" in g else None
    stream = _routes(lambda: st.push(x[..., :3 * st.hop], None, gid))
    assert len(whole) == len(m.encoder.layers)
    # the stream's launches: the encoder's layers, then the local embedding (none here) and the decoder's
    enc = stream[:len(whole)]
    norm = lambda r: r if r[0] == "ffma" else ("tc",)  # noqa: E731 - the tile height follows the launch's length
    assert [norm(r) for r in enc] == [norm(r) for r in whole], (enc, whole)
    assert any(r[0] == "tc" for r in whole) if name == "vqvae_vctk_g" else True


# ---------------------------------------------------------------------------------------------------- end to end
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("sched", list(SCHEDULES))
def test_stream_equals_decode_encode(dev, name, sched):
    from parallelwavegan_b200.streaming import VQVAELookaheadStream

    meta, g, m = _model(dev, name)
    x = g["x"].to(dev)
    l = g["l"].to(dev) if "l" in g else None
    gid = g["g"].to(dev) if "g" in g else None
    st = VQVAELookaheadStream(m, batch=x.shape[0], use_graphs=sched != "ones")
    _check(m, st, x, l, gid, SCHEDULES[sched])
    _check(m, st, x, l, gid, SCHEDULES[sched])  # the flush left every slot fresh


@pytest.mark.parametrize("name", ["vqvae_yesno", "vqvae_vctk_lg"])
def test_without_weight_norm(dev, name):
    from parallelwavegan_b200.streaming import VQVAELookaheadStream

    meta, g, m = _model(dev, name, weight_norm=False)
    x = g["x"].to(dev)
    l = g["l"].to(dev) if "l" in g else None
    gid = g["g"].to(dev) if "g" in g else None
    _check(m, VQVAELookaheadStream(m, batch=x.shape[0]), x, l, gid, [2, 5])


def test_delay_and_plan(dev):
    from parallelwavegan_b200.streaming import MelGANLookaheadStream, VQVAELookaheadStream

    for name in NAMES:
        _, g, m = _model(dev, name)
        st = VQVAELookaheadStream(m, batch=1)
        assert st.E == 12 and st.hop == 64 and st.delay == 12 * 64 + st.dec_delay
        assert st.dec_delay == MelGANLookaheadStream(m.decoder).delay and st.min_frames == MelGANLookaheadStream(m.decoder).min_frames


def test_four_slots_speakers_reset_and_partial_flush(dev):
    """four slots converting to different speakers; slot 1 is reset mid-stream and restarts with another signal and
    speaker; slot 2 is flushed while the others continue unchanged; graphs and eager give the same samples"""
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import VQVAELookaheadStream

    _, g, m = _model(dev, "vqvae_vctk_lg")
    B, T, hop = 4, 20, 64
    xs = [synth.randn((1, T * hop), 500 + k, 0.5).to(dev) for k in range(B + 1)]
    ls = [synth.randn((1, 2, T), 600 + k).to(dev) for k in range(B + 1)]

    def ref(k, frames, spk):
        return _reference(m, xs[k][:, None, :frames * hop], ls[k][..., :frames], torch.tensor([spk], device=dev))[1][0, 0]

    outs = {}
    for graphs in (True, False):
        st = VQVAELookaheadStream(m, batch=B, use_graphs=graphs)
        sig, pos, spk = [0, 1, 2, 3], [0] * B, [3, 50, 7, 99]
        got = {b: [] for b in range(B)}

        def push(n):
            x = torch.cat([xs[sig[b]][:, pos[b] * hop:(pos[b] + n) * hop] for b in range(B)])
            l = torch.cat([ls[sig[b]][..., pos[b]:pos[b] + n] for b in range(B)])
            y = st.push(x, l, torch.tensor(spk, device=dev))
            for b in range(B):
                pos[b] += n
                got[b].append(y[b, 0])

        push(5)
        st.reset(1)
        sig[1], pos[1], spk[1], got[1] = 4, 0, 11, []
        with pytest.raises(PwgbError):  # slot 2 may not change speaker inside its signal
            st.push(torch.zeros(B, hop, device=dev), torch.zeros(B, 2, 1, device=dev), torch.tensor([3, 11, 8, 99], device=dev))
        push(5)
        tail2 = st.flush(2)[0, 0]
        full2 = torch.cat(got[2] + [tail2])
        assert torch.equal(full2, torch.cat([torch.zeros(st.delay, device=dev), ref(2, 10, 7)]))
        sig[2], pos[2], got[2] = 2, 0, []
        push(5)
        push(5)
        tail = st.flush([0, 1, 3])
        full = {b: torch.cat(got[b] + [tail[i, 0]]) for i, b in enumerate([0, 1, 3])}
        z = torch.zeros(st.delay, device=dev)
        assert torch.equal(full[0], torch.cat([z, ref(0, 20, 3)]))
        assert torch.equal(full[1], torch.cat([z, ref(4, 15, 11)]))
        assert torch.equal(full[3], torch.cat([z, ref(3, 20, 99)]))
        outs[graphs] = (full[0], full[1], full2, full[3])
    assert all(torch.equal(a, b) for a, b in zip(outs[True], outs[False]))


def _gaps(z_e, cb):
    """fp64 (best-to-second gap / distance scale) of every frame, as the goldens' codebook scale was chosen"""
    x = z_e.double().transpose(1, 2).reshape(-1, cb.shape[1])
    c = cb.double()
    d = (c * c).sum(1)[None] + (x * x).sum(1)[:, None] - 2 * x @ c.t()
    s = d.sort(dim=1)[0]
    return (s[:, 1] - s[:, 0]) / ((x * x).sum(1) + (c * c).sum(1).max())


def test_long_signal_codes_and_rel_l2(dev):
    """beyond 4096 samples the whole utterance's output conv changes kernel: the codes stay equal (on frames whose
    best-to-second gap is at least 1e-3 of the distance scale) and the output agrees to rel-L2 1e-6"""
    from parallelwavegan_b200.streaming import VQVAELookaheadStream

    _, g, m = _model(dev, "vqvae_vctk_g")
    T = 150
    x = synth.randn((2, 1, T * 64), 77, 0.5).to(dev)
    gid = torch.tensor([4, 90], device=dev)
    ref_idx, ref = _reference(m, x, None, gid)
    st = VQVAELookaheadStream(m, batch=2)
    y, idx = _stream(st, x, None, gid, [1, 4, 2, 9, 1, 3])
    with torch.no_grad():
        gap = _gaps(m.encoder(x)[-1].cpu(), m.codebook.embedding.weight.detach().cpu()).reshape(2, T)
    clear = gap >= 1e-3
    assert len(set(ref_idx.cpu()[clear].tolist())) >= 8
    assert torch.equal(idx.cpu()[clear], ref_idx.cpu()[clear])
    assert rel_l2(y[..., st.delay:].cpu(), ref.cpu()) <= 1e-6


def test_state_bytes(dev):
    from parallelwavegan_b200.streaming import VQVAELookaheadStream

    _, _, m = _model(dev, "vqvae_vctk_lg")
    st = VQVAELookaheadStream(m, batch=2)
    n = sum(t.numel() * t.element_size() for t in st._state()) // 2
    assert st.state_bytes() == n and st.l_hist.shape == (2, 32, 12)


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals_before_any_launch(dev):
    from parallelwavegan_b200 import capi, models
    from parallelwavegan_b200.capi import PwgbError
    from parallelwavegan_b200.streaming import VQVAELookaheadStream

    meta, g, m = _model(dev, "vqvae_yesno")
    kw = copy.deepcopy(meta["kwargs"])
    cpu = _model(dev, "vqvae_yesno")[2].cpu()
    bad = [models.MelGANGenerator(in_channels=8, channels=64, upsample_scales=[4, 4, 2, 2], stacks=2),
           models.VQVAE(**dict(kw, encoder_type="ParallelWaveGANDiscriminator", encoder_conf={"out_channels": 8})),
           models.VQVAE(**dict(kw, decoder_conf=dict(kw["decoder_conf"], use_causal_conv=True))),
           models.VQVAE(**dict(kw, decoder_conf=dict(kw["decoder_conf"], upsample_scales=[4, 4, 2]))),
           models.VQVAE(**dict(kw, in_channels=2)),
           m.train(), cpu]
    torch.cuda.synchronize()
    capi.reset_launch_count()
    for i, mm in enumerate(bad):
        if i < 5:
            mm = mm.to(dev).eval()
        with pytest.raises(PwgbError):
            VQVAELookaheadStream(mm)
    m.eval()
    st = VQVAELookaheadStream(m, batch=2)
    for args in ((torch.zeros(2, 100, device=dev),), (torch.zeros(2, 0, device=dev),), (torch.zeros(3, 64, device=dev),),
                 (torch.zeros(2, 64, device=dev), torch.zeros(2, 2, 1, device=dev)),
                 (torch.zeros(2, 64, device=dev), None, torch.tensor([0, 1], device=dev))):
        with pytest.raises(PwgbError):
            st.push(*args)
    with pytest.raises(PwgbError):
        st.flush()  # no frames yet: decode needs min_frames
    assert capi.launch_count() == 0
    _, g2, m2 = _model(dev, "vqvae_vctk_lg")
    st2 = VQVAELookaheadStream(m2, batch=2)
    capi.reset_launch_count()
    with pytest.raises(PwgbError):
        st2.push(torch.zeros(2, 64, device=dev), None, torch.tensor([0, 1], device=dev))  # l required
    with pytest.raises(PwgbError):
        st2.push(torch.zeros(2, 64, device=dev), torch.zeros(2, 2, 1, device=dev))  # g required
    assert capi.launch_count() == 0
