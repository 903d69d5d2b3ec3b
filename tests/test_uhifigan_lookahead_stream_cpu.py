"""Streaming a centred U-Net HiFi-GAN with a fixed lookahead, on the CPU: the chunked oracle
(oracle/ref_uhifigan_lookahead_stream.py) followed by its flush equals [zeros(delay) | the whole-utterance generator]
in float64 for every chunk schedule and for utterances shorter than the delay, its delay is the lookahead autograd
measures at every output phase, and each plausible mistake breaks that equality."""
import pytest
import torch

from helpers import golden_effective_weights, load_golden
from oracle import ref_uhifigan_lookahead_stream as RU
from oracle import synth

# one frame at a time, 3 frames, 7 frames and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
TOL = 1e-12
YESNO = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, downsample_scales=[2, 2, 8, 8],
             downsample_kernel_sizes=[4, 4, 16, 16], upsample_scales=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4],
             resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3, use_additional_convs=True, bias=True)


def _setup(name, frames=None):
    """(cfg, float64 effective weights, e (B, 1, T * hop), c (B, 80, T)) of a golden model, or of the yesno recipe's
    shape with synthetic weights (``yesno``)"""
    if name == "yesno":
        from parallelwavegan_b200 import models
        from oracle.ref_ops import fold_weight_norm

        m = models.UHiFiGANGenerator(**YESNO)
        sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, 1.15)
        T = frames or 3
        return YESNO, {k: v.double() for k, v in fold_weight_norm(sd).items()}, synth.randn((1, 1, T * 256), 33, 0.3).double(), \
            synth.randn((1, 80, T), 32).double()
    meta, _ = load_golden(name)
    w = golden_effective_weights(meta)
    c = synth.randn(meta["c_shape"], meta["c_seed"]).double()
    e = synth.randn(meta["e_shape"], meta["e_seed"], meta["e_scale"]).double()
    if frames:
        c, e = c[..., :frames], e[..., :frames * meta["hop"]]
    return meta["kwargs"], {k: v.double() for k, v in w.items()}, e, c


def _expected(w, e, c, cfg, delay):
    ref = RU.whole_utterance(w, e, c, cfg)
    return torch.cat([ref.new_zeros(ref.shape[:-1] + (delay,)), ref], -1)


def _err(y, ref):
    return float((y - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("name", ["uhifigan_small", "uhifigan_odd", "uhifigan_opencpop"])
def test_chunked_oracle_equals_whole_utterance(name, schedule):
    cfg, w, e, c = _setup(name)
    delay = RU.UHiFiGANLookaheadRef(w, cfg).delay
    ref = _expected(w, e, c, cfg, delay)
    y = RU.stream(w, e, c, cfg, SCHEDULES[schedule])
    assert y.shape == ref.shape
    assert _err(y, ref) <= TOL, _err(y, ref)


@pytest.mark.parametrize("frames", [1, 2, 5])
@pytest.mark.parametrize("name", ["uhifigan_small", "uhifigan_odd", "uhifigan_opencpop"])
def test_utterances_shorter_than_the_delay(name, frames):
    """the audio of an utterance shorter than the delay comes almost entirely from the flush"""
    cfg, w, e, c = _setup(name, frames)
    ref = RU.UHiFiGANLookaheadRef(w, cfg)
    assert frames * ref.hop < ref.delay
    expected = _expected(w, e, c, cfg, ref.delay)
    for schedule in (SCHEDULES["ones"], SCHEDULES["long"]):
        assert _err(RU.stream(w, e, c, cfg, schedule), expected) <= TOL


@pytest.mark.parametrize("name, delay, e_look", [("uhifigan_odd", 83, 86), ("uhifigan_small", 1846, 1851),
                                                 ("uhifigan_opencpop", 16231, 16455), ("yesno", 5050, 5235)])
def test_delay_is_the_measured_lookahead(name, delay, e_look):
    """``delay`` equals the largest lookahead autograd measures over the output phases of one hop, with no excess: the
    last frame an output needs, times hop, minus the output's index.  The excitation-sample lookahead (the last
    excitation sample an output reads, minus its index) is larger by up to hop - 1 at some phases, but that sample
    arrives with its whole frame, so it does not bound the delay of a stream fed frame by frame."""
    cfg, w, _, _ = _setup(name)
    ref = RU.UHiFiGANLookaheadRef(w, cfg)
    assert ref.delay == delay
    hop = ref.hop
    phases = RU.measured_lookahead(w, cfg, 2 + delay // hop + 4)
    assert len(phases) == hop
    assert max(f for _, f in phases) == delay
    assert all(delay >= f for _, f in phases)
    assert max(k for k, _ in phases) == e_look


def test_opencpop_plan():
    """the per-level lookaheads and delay lines of the opencpop recipe (DESIGN.md §3.11)"""
    cfg, w, _, _ = _setup("uhifigan_opencpop")
    ref = RU.UHiFiGANLookaheadRef(w, cfg)
    assert [(lv["look_in"], lv["look"], lv["H"]) for lv in ref.enc] == [(63, 13, 5), (73, 15, 5), (75, 20, 7), (80, 27, 3)]
    assert ref.look_dec0 == 27 and ref.cin_len == 30
    assert [(lv["d1"], lv["d2"], lv["look_u"]) for lv in ref.dec] == [(0, 0, 83), (0, 123, 574), (0, 619, 3173), (0, 3220, 16168)]


MISTAKES = ["skip_undelayed", "mel_undelayed", "stride_phase", "ds_no_end_mask", "s2d_no_hist"]


@pytest.mark.parametrize("mistake", MISTAKES)
@pytest.mark.parametrize("name", ["uhifigan_small", "uhifigan_odd"])
def test_mistakes_are_caught(name, mistake):
    """each mistake moves the output by many orders of magnitude more than the tolerance (the odd config's mel path and
    deepest skip share a lookahead, so there the mel path has no delay to forget)"""
    cfg, w, e, c = _setup(name)
    ref = RU.UHiFiGANLookaheadRef(w, cfg)
    if mistake == "mel_undelayed" and ref.cin_len == cfg["kernel_size"] - 1:
        pytest.skip("the mel path is not delayed in this config")
    expected = _expected(w, e, c, cfg, ref.delay)
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        assert _err(RU.stream(w, e, c, cfg, schedule), expected) <= TOL
        assert _err(RU.stream(w, e, c, cfg, schedule, **{mistake: True}), expected) > 1e6 * TOL, (mistake, schedule)
