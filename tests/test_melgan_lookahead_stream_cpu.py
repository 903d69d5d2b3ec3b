"""Streaming a centred (multi-band) MelGAN with a fixed lookahead, on the CPU: the chunked oracle
(oracle/ref_melgan_lookahead_stream.py) followed by its flush equals [zeros(delay) | the whole-utterance centred generator]
in float64 for every chunk schedule, all three pads, with and without PQMF and at the shortest utterance ``inference``
accepts; it reproduces the golden ``inference`` outputs of the real reference; its delay is the lookahead autograd
measures; and each plausible mistake breaks that equality."""
import json

import pytest
import torch

from helpers import ORACLE_TOL, golden_effective_weights, load_golden, rel_l2
from oracle import ref_melgan_lookahead_stream as RL
from oracle import synth
from oracle.ref_ops import fold_weight_norm

# one frame at a time (from a fresh slot), 3 frames, 7 frames and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
TOL = 1e-12
PADS = {"reflect": {}, "replicate": dict(pad="ReplicationPad1d"), "zero": dict(pad="ConstantPad1d", pad_params={"value": 0.0})}
V1 = dict(in_channels=80, out_channels=1, kernel_size=7, channels=512, upsample_scales=[8, 8, 2, 2], stack_kernel_size=3, stacks=3)
MB_V2 = dict(in_channels=80, out_channels=4, kernel_size=7, channels=384, upsample_scales=[8, 4, 2], stack_kernel_size=3, stacks=4)
# the golden centred models (reflect full-band without tanh, replicate, zero, reflect multi-band at [5, 5, 3] and at
# [3, 4, 2]) and synthetic multi-band models with the other pads
GOLDEN = ["melgan_small", "melgan_centred_replicate", "melgan_centred_zero", "mb_melgan_v2", "melgan_centred_mb"]
SYNTH = {
    "mb_replicate": dict(MB_V2, channels=32, upsample_scales=[4, 2], stacks=3, **PADS["replicate"]),
    "mb_zero_relu": dict(MB_V2, channels=32, upsample_scales=[3, 5], stacks=2, nonlinear_activation="ReLU", nonlinear_activation_params={},
                         **PADS["zero"]),
}


def _cfg(kw):
    slope = 0.0 if kw.get("nonlinear_activation") == "ReLU" else kw.get("nonlinear_activation_params", {}).get("negative_slope", 0.2)
    pad = {"ReflectionPad1d": "reflect", "ReplicationPad1d": "replicate", "ConstantPad1d": "zero"}[kw.get("pad", "ReflectionPad1d")]
    return dict(kw, negative_slope=slope), pad, (kw["out_channels"] if kw["out_channels"] > 1 else None)


def _setup(name, frames=None):
    """(cfg, pad, subbands, float64 effective weights, c (B, 80, T) float64)"""
    if name in SYNTH or name in ("v1_256", "mb_v2_128", "mb_v2_csmsc_128"):
        from parallelwavegan_b200 import models

        kw = SYNTH.get(name) or dict(V1 if name == "v1_256" else MB_V2, channels=int(name.rsplit("_", 1)[1]))
        if name == "mb_v2_csmsc_128":
            kw["upsample_scales"] = [5, 5, 3]
        m = models.MelGANGenerator(**json.loads(json.dumps(kw)))
        sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 33, 1.0)
        c = synth.randn((2, 80, frames or 13), 34).double()
        return (*_cfg(kw), {k: v.double() for k, v in fold_weight_norm(sd).items()}, c)
    meta, _ = load_golden(name)
    w = golden_effective_weights(meta)
    c = synth.randn(meta["c_shape"], meta["c_seed"]).double()
    return (*_cfg(meta["kwargs"]), {k: v.double() for k, v in w.items()}, c[..., :frames] if frames else c)


def _expected(w, c, cfg, pad, sb):
    delay = RL.MelGANLookaheadRef(w, cfg, pad, sb).delay
    ref = RL.whole_utterance(w, c, cfg, pad, sb)
    return torch.cat([ref.new_zeros(ref.shape[:-1] + (delay,)), ref], -1)


def _err(y, ref):
    return float((y - ref).abs().max() / ref.abs().max())


def test_min_frames_of_the_recipes():
    assert RL.min_frames(V1) == RL.min_frames(MB_V2) == 4
    assert RL.min_frames(dict(MB_V2, upsample_scales=[5, 5, 3])) == 6
    assert RL.min_frames(V1, "replicate") == RL.min_frames(MB_V2, "zero") == 1


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("name", GOLDEN + list(SYNTH))
def test_chunked_oracle_equals_whole_utterance(name, schedule):
    cfg, pad, sb, w, c = _setup(name)
    ref = _expected(w, c, cfg, pad, sb)
    y = RL.stream(w, c, cfg, SCHEDULES[schedule], pad, sb)
    assert y.shape == ref.shape
    assert _err(y, ref) <= TOL, _err(y, ref)


@pytest.mark.parametrize("name", GOLDEN + list(SYNTH))
def test_shortest_utterance(name):
    """at the shortest length ``inference`` accepts, the audio comes mostly from the flush"""
    cfg, pad, sb, w, c = _setup(name)
    c = c[..., :RL.min_frames(cfg, pad)]
    ref = _expected(w, c, cfg, pad, sb)
    for schedule in (SCHEDULES["ones"], SCHEDULES["long"]):
        assert _err(RL.stream(w, c, cfg, schedule, pad, sb), ref) <= TOL


@pytest.mark.parametrize("name", ["melgan_small", "melgan_centred_replicate", "melgan_centred_zero", "mb_melgan_v2", "melgan_centred_mb"])
def test_chunked_oracle_reproduces_golden_inference(name):
    meta, g = load_golden(name)
    cfg, pad, sb, w, c = _setup(name)
    delay = RL.MelGANLookaheadRef(w, cfg, pad, sb).delay
    y = RL.stream({k: v.float() for k, v in w.items()}, c[:1].float(), cfg, SCHEDULES["mixed"], pad, sb, dtype=torch.float32)
    # melgan_small stores the forward of both utterances, which for a full-band model is inference
    assert rel_l2(y[0, :, delay:].t(), g["y_inf"] if "y_inf" in g else g["y"][0].t()) < ORACLE_TOL


@pytest.mark.parametrize("name, pad, delay", [("v1_256", "reflect", 1425), ("mb_v2_128", "reflect", 4 * 672 + 31),
                                              ("mb_v2_csmsc_128", "reflect", 4 * 1044 + 31), ("melgan_small", "reflect", 81),
                                              ("melgan_centred_mb", "reflect", None)])
def test_delay_is_the_measured_lookahead(name, pad, delay):
    """the padding sum is tight: autograd on the float64 model measures the same lookahead"""
    cfg, pad, sb, w, _ = _setup(name)
    ref = RL.MelGANLookaheadRef(w, cfg, pad, sb)
    if delay is not None:
        assert ref.delay == delay
    hop = ref.hop * (sb or 1)
    frames = max(-(-ref.delay // hop) + 3, RL.min_frames(cfg, pad) + 1)
    assert RL.measured_lookahead(w, cfg, frames, pad, sb) == ref.delay


MISTAKES = ["zero_edges", "left_only", "wrong_axis", "undelayed_skip", "unmasked_pqmf", "flush_no_end"]


@pytest.mark.parametrize("name, mistake", [("melgan_centred_mb", m) for m in MISTAKES] +
                         [("melgan_small", m) for m in MISTAKES if m != "unmasked_pqmf"])
def test_mistakes_are_caught(name, mistake):
    """each mistake moves the output by many orders of magnitude more than the tolerance (a full-band model has no PQMF
    output to mask)"""
    cfg, pad, sb, w, c = _setup(name)
    ref = _expected(w, c, cfg, pad, sb)
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        assert _err(RL.stream(w, c, cfg, schedule, pad, sb), ref) <= TOL
        assert _err(RL.stream(w, c, cfg, schedule, pad, sb, **{mistake: True}), ref) > 1e6 * TOL, (mistake, schedule)


@pytest.mark.parametrize("mistake", ["zero_edges", "left_only"])
def test_replicate_mistakes_are_caught(mistake):
    cfg, pad, sb, w, c = _setup("melgan_centred_replicate")
    ref = _expected(w, c, cfg, pad, sb)
    assert _err(RL.stream(w, c, cfg, SCHEDULES["short"], pad, sb), ref) <= TOL
    assert _err(RL.stream(w, c, cfg, SCHEDULES["short"], pad, sb, **{mistake: True}), ref) > 1e6 * TOL
