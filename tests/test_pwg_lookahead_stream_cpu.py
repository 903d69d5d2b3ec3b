"""Streaming a centred Parallel WaveGAN with a fixed lookahead, on the CPU: the chunked oracle
(oracle/ref_pwg_lookahead_stream.py) followed by its flush equals [zeros(delay) | the whole-utterance centred generator]
in float64 for every chunk schedule and for utterances shorter than the delay, its delay is the lookahead autograd
measures, and each plausible mistake breaks that equality."""
import pytest
import torch

from helpers import golden_effective_weights, load_golden
from oracle import ref_pwg_lookahead_stream as RL
from oracle import synth

# one frame at a time, 3 frames, 7 frames and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
TOL = 1e-12


def _setup(name, frames=None):
    """(cfg, float64 effective weights, z (B, 1, T * hop), c (B, aux, T)) of a centred PWG golden model"""
    meta, _ = load_golden(name)
    kw = meta["kwargs"]
    cfg = dict(kw, upsample_scales=kw["upsample_params"]["upsample_scales"])
    w = {k: v.double() for k, v in golden_effective_weights(meta).items()}
    ctx = kw["aux_context_window"]
    c = synth.randn(meta["c_shape"], meta["c_seed"]).double()
    c = c[:, :, ctx:c.shape[-1] - ctx]
    z = synth.randn(meta["z_shape"], meta["z_seed"]).double()
    if frames:
        hop = z.shape[-1] // c.shape[-1]
        c, z = c[..., :frames], z[..., :frames * hop]
    return cfg, w, z, c


def _expected(w, z, c, cfg, delay):
    ref = RL.whole_utterance(w, z, c, cfg)
    return torch.cat([ref.new_zeros(ref.shape[:-1] + (delay,)), ref], -1)


def _err(y, ref):
    return float((y - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("name", ["pwg_small", "pwg_v1"])
def test_chunked_oracle_equals_whole_utterance(name, schedule):
    cfg, w, z, c = _setup(name)
    delay = RL.plan(cfg)[-1]
    ref = _expected(w, z, c, cfg, delay)
    y = RL.stream(w, z, c, cfg, SCHEDULES[schedule])
    assert y.shape == ref.shape
    assert _err(y, ref) <= TOL, _err(y, ref)


@pytest.mark.parametrize("name, frames", [("pwg_small", 1), ("pwg_v1", 1), ("pwg_v1", 2), ("pwg_v1", 5)])
def test_utterances_shorter_than_the_delay(name, frames):
    """the audio of an utterance shorter than the delay comes almost entirely from the flush"""
    cfg, w, z, c = _setup(name, frames)
    delay = RL.plan(cfg)[-1]
    assert frames * RL.PWGLookaheadRef(w, cfg).hop < delay
    ref = _expected(w, z, c, cfg, delay)
    for schedule in (SCHEDULES["ones"], SCHEDULES["long"]):
        assert _err(RL.stream(w, z, c, cfg, schedule), ref) <= TOL


@pytest.mark.parametrize("name, look_c, look_x, delay", [("pwg_v1", 852, 851, 3920), ("pwg_small", 20, 19, 28)])
def test_delay_is_the_measured_lookahead(name, look_c, look_x, delay):
    """the plan is tight: autograd finds exactly that lookahead on the whole-utterance model.  The conditioning enters
    layer 0 after its dilated conv, so the delay is (kernel - 1) / 2 * d_0 short of look_c + D_L"""
    cfg, w, _, _ = _setup(name)
    _, looks, lx, D, d = RL.plan(cfg)
    assert (looks[-1], lx, d) == (look_c, look_x, delay)
    assert d == look_c + D[-1] - D[0]
    ref = RL.PWGLookaheadRef(w, cfg)
    assert ref.delay == delay
    frames = -(-delay // ref.hop) + 3
    assert RL.measured_lookahead(w, cfg, frames) == delay


MISTAKES = ["no_mask", "undelayed_res", "unaligned_skips", "undelayed_cond", "undelayed_noise", "flush_zero_edge"]


@pytest.mark.parametrize("mistake", MISTAKES)
@pytest.mark.parametrize("name", ["pwg_small", "pwg_v1"])
def test_mistakes_are_caught(name, mistake):
    """each mistake moves the output by many orders of magnitude more than the tolerance.  pwg_small has no conv_in
    context (acw 0), so its flush has no replicated edge to get wrong."""
    if mistake == "flush_zero_edge" and name == "pwg_small":
        pytest.skip("acw 0: the flush pushes no replicated frame")
    cfg, w, z, c = _setup(name)
    delay = RL.plan(cfg)[-1]
    ref = _expected(w, z, c, cfg, delay)
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        assert _err(RL.stream(w, z, c, cfg, schedule), ref) <= TOL
        assert _err(RL.stream(w, z, c, cfg, schedule, **{mistake: True}), ref) > 1e6 * TOL, (mistake, schedule)
