"""Streaming a centred HiFi-GAN with a fixed lookahead, on the CPU: the chunked oracle
(oracle/ref_hifigan_lookahead_stream.py) followed by its flush equals [zeros(delay) | the whole-utterance centred
generator] in float64 for every chunk schedule and for utterances shorter than the delay, its delay is the lookahead
autograd measures, and each plausible mistake breaks that equality."""
import json

import pytest
import torch

from helpers import golden_effective_weights, load_golden
from oracle import ref_hifigan_lookahead_stream as RL
from oracle import synth
from oracle.ref_ops import fold_weight_norm

# one frame at a time, 3 frames, longer than the input conv's 6-frame history, and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
TOL = 1e-12
V1 = dict(in_channels=80, out_channels=1, channels=512, kernel_size=7, upsample_scales=[8, 8, 2, 2],
          upsample_kernel_sizes=[16, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3)


def _cfg(kw):
    slope = 0.0 if kw.get("nonlinear_activation") == "ReLU" else kw.get("nonlinear_activation_params", {}).get("negative_slope", 0.1)
    return dict(kw, negative_slope=slope)


def _setup(name, frames=None):
    """(cfg, float64 effective weights, c (B, 80, T) float64) of a golden model, or of a v1-shaped synthetic model with
    ``channels`` channels (``v1_<channels>``)"""
    if name.startswith("v1_"):
        from parallelwavegan_b200 import models

        kw = dict(V1, channels=int(name[3:]))
        m = models.HiFiGANGenerator(**json.loads(json.dumps(kw)))
        sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 23, 1.15)
        return _cfg(kw), {k: v.double() for k, v in fold_weight_norm(sd).items()}, synth.randn((1, 80, frames or 9), 24).double()
    meta, _ = load_golden(name)
    w = golden_effective_weights(meta)
    c = synth.randn(meta["c_shape"], meta["c_seed"]).double()
    return _cfg(meta["kwargs"]), {k: v.double() for k, v in w.items()}, c[..., :frames] if frames else c


def _expected(w, c, cfg, delay):
    ref = RL.whole_utterance(w, c, cfg)
    return torch.cat([ref.new_zeros(ref.shape[:-1] + (delay,)), ref], -1)


def _err(y, ref):
    return float((y - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("name", ["hifigan_small", "hifigan_odd", "hifigan_v1"])
def test_chunked_oracle_equals_whole_utterance(name, schedule):
    cfg, w, c = _setup(name)
    delay = RL.HiFiGANLookaheadRef(w, cfg).delay
    ref = _expected(w, c, cfg, delay)
    y = RL.stream(w, c, cfg, SCHEDULES[schedule])
    assert y.shape == ref.shape
    assert _err(y, ref) <= TOL, _err(y, ref)


@pytest.mark.parametrize("frames", [1, 2, 5])
@pytest.mark.parametrize("name", ["hifigan_odd", "v1_16"])
def test_utterances_shorter_than_the_delay(name, frames):
    """the audio of an utterance shorter than the delay comes almost entirely from the flush"""
    cfg, w, c = _setup(name, frames)
    delay = RL.HiFiGANLookaheadRef(w, cfg).delay
    assert frames * RL.HiFiGANLookaheadRef(w, cfg).hop < delay
    ref = _expected(w, c, cfg, delay)
    for schedule in (SCHEDULES["ones"], SCHEDULES["long"]):
        assert _err(RL.stream(w, c, cfg, schedule), ref) <= TOL


@pytest.mark.parametrize("name, delay", [("v1_16", 3258), ("hifigan_odd", 170)])
def test_delay_is_the_measured_lookahead(name, delay):
    cfg, w, _ = _setup(name)
    ref = RL.HiFiGANLookaheadRef(w, cfg)
    assert ref.delay == delay
    frames = -(-delay // ref.hop) + 3
    assert RL.measured_lookahead(w, cfg, frames) == delay


@pytest.mark.parametrize("mistake", ["no_mask", "undelayed_res", "unaligned", "flush_no_end"])
@pytest.mark.parametrize("name", ["hifigan_small", "hifigan_odd"])
def test_mistakes_are_caught(name, mistake):
    """each mistake moves the output by many orders of magnitude more than the tolerance"""
    cfg, w, c = _setup(name)
    delay = RL.HiFiGANLookaheadRef(w, cfg).delay
    ref = _expected(w, c, cfg, delay)
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        assert _err(RL.stream(w, c, cfg, schedule), ref) <= TOL
        assert _err(RL.stream(w, c, cfg, schedule, **{mistake: True}), ref) > 1e6 * TOL, (mistake, schedule)


@pytest.mark.parametrize("name", ["hifigan_small", "hifigan_odd"])
def test_conv_transpose_history_only_reaches_masked_samples(name):
    """a fresh slot's conv-transpose history is level-input sample -(look + 1), look >= 3 being the lookahead of the level
    input, and its taps reach only output samples before 0, which the mask zeroes: replicating the signal's sample 0
    there, as the causal model's ReplicationPad1d does, changes nothing, and the stream passes no replicate flags.  So a
    replicated history is not a mistake the output can show; this test shows it is masked instead.  The first push holds
    the whole utterance, so that it reaches sample 0 of every level input."""
    cfg, w, c = _setup(name)
    delay = RL.HiFiGANLookaheadRef(w, cfg).delay
    ref = _expected(w, c, cfg, delay)
    whole = [c.shape[-1]]
    assert _err(RL.stream(w, c, cfg, whole, up_replicate=True), ref) <= TOL
    assert _err(RL.stream(w, c, cfg, whole, up_replicate=True, no_mask=True), ref) > 1e6 * TOL
