"""Streaming a causal (multi-band) MelGAN, on the CPU: the chunked oracle (oracle/ref_melgan_stream.py) equals the
whole-utterance causal generator in float64, after the PQMF delay, for every chunk schedule, all three pads and with and
without PQMF; it reproduces the golden ``inference`` outputs of the real reference; and each plausible state mistake
breaks that equality."""
import json

import pytest
import torch
import torch.nn.functional as F

from helpers import ORACLE_TOL, golden_effective_weights, load_golden, rel_l2
from oracle import ref_melgan_stream as RS
from oracle import synth
from oracle.ref_ops import fold_weight_norm

# after the opening push: one frame at a time, 3 frames, and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "mixed": [1, 4, 2, 9, 1, 3]}
TOL = 1e-12
PADS = {"reflect": {}, "replicate": dict(pad="ReplicationPad1d"), "zero": dict(pad="ConstantPad1d", pad_params={"value": 0.0})}
SMALL_MB = dict(in_channels=80, out_channels=4, kernel_size=7, channels=64, upsample_scales=[4, 4, 2], stack_kernel_size=3, stacks=3,
                use_causal_conv=True)
# the golden fixtures (reflect full-band, replicate full-band, zero full-band, reflect multi-band) and synthetic
# multi-band models with the two other pads and ReLU
CASES = {
    "melgan_causal": None, "melgan_causal_replicate": None, "melgan_causal_zero": None, "melgan_causal_mb": None,
    "mb_replicate": dict(SMALL_MB, **PADS["replicate"]),
    "mb_zero_relu": dict(SMALL_MB, upsample_scales=[3, 5], stacks=2, nonlinear_activation="ReLU", nonlinear_activation_params={},
                         **PADS["zero"]),
}


def _cfg(kw):
    slope = 0.0 if kw.get("nonlinear_activation") == "ReLU" else kw.get("nonlinear_activation_params", {}).get("negative_slope", 0.2)
    pad = {"ReflectionPad1d": "reflect", "ReplicationPad1d": "replicate", "ConstantPad1d": "zero"}[kw.get("pad", "ReflectionPad1d")]
    return dict(kw, negative_slope=slope), pad, (kw["out_channels"] if kw["out_channels"] > 1 else None)


def _setup(name):
    """(cfg, pad, subbands, float64 effective weights, c (2, 80, T) float64)"""
    kw = CASES[name]
    if kw is None:
        meta, _ = load_golden(name)
        w = golden_effective_weights(meta)
        return (*_cfg(meta["kwargs"]), {k: v.double() for k, v in w.items()}, synth.randn(meta["c_shape"], meta["c_seed"]).double())
    from parallelwavegan_b200 import models

    m = models.MelGANGenerator(**json.loads(json.dumps(kw)))
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, 1.0)
    return (*_cfg(kw), {k: v.double() for k, v in fold_weight_norm(sd).items()}, synth.randn((2, 80, 17), 32).double())


def min_first_frames(cfg, pad):
    """max over the reflect-padded convs of floor(P / rate) + 1 (1 for the other pads)"""
    if pad != "reflect":
        return 1
    need, rate = [(cfg["kernel_size"] - 1, 1)], 1
    for s in cfg["upsample_scales"]:
        rate *= s
        need += [((cfg.get("stack_kernel_size", 3) - 1) * cfg.get("stack_kernel_size", 3) ** j, rate) for j in range(cfg["stacks"])]
    need.append((cfg["kernel_size"] - 1, rate))
    return max(P // r + 1 for P, r in need)


def _delayed(ref, subbands):
    """[zeros(taps // 2) | whole utterance]: what the stream's pushes and flush concatenate to"""
    return F.pad(ref, (31, 0)) if subbands else ref


def _err(y, ref):
    return float((y - ref).abs().max() / ref.abs().max())


def test_min_first_frames_of_the_recipes():
    v1 = dict(kernel_size=7, upsample_scales=[8, 8, 2, 2], stacks=3)
    mb2 = dict(kernel_size=7, upsample_scales=[8, 4, 2], stacks=4)
    assert min_first_frames(v1, "reflect") == min_first_frames(mb2, "reflect") == 7
    assert min_first_frames(v1, "replicate") == min_first_frames(mb2, "zero") == 1


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("name", list(CASES))
def test_chunked_oracle_equals_whole_utterance(name, schedule):
    cfg, pad, sb, w, c = _setup(name)
    ref = _delayed(RS.whole_utterance(w, c, cfg, pad, sb), sb)
    y = RS.stream(w, c, cfg, SCHEDULES[schedule], pad, sb, first=min_first_frames(cfg, pad))
    assert y.shape == ref.shape
    assert _err(y, ref) <= TOL, _err(y, ref)


@pytest.mark.parametrize("name", ["melgan_causal", "melgan_causal_replicate", "melgan_causal_zero", "melgan_causal_mb"])
def test_chunked_oracle_reproduces_golden_inference(name):
    meta, g = load_golden(name)
    cfg, pad, sb, w, c = _setup(name)
    y = RS.stream({k: v.float() for k, v in w.items()}, c[:1].float(), cfg, SCHEDULES["mixed"], pad, sb,
                  first=min_first_frames(cfg, pad), dtype=torch.float32)
    y = y[0, :, 31:] if sb else y[0]
    # melgan_causal stores the forward of both utterances, which for a full-band model is inference
    assert rel_l2(y.t(), g["y_inf"] if "y_inf" in g else g["y"][0].t()) < ORACLE_TOL


MISTAKES = {"stack_short": dict(stack_short=1), "fresh_zero": dict(fresh_zero=True), "up_zero": dict(up_zero=True),
            "pq_short": dict(pq_short=1), "flush_edge": dict(flush_edge=True)}


@pytest.mark.parametrize("mistake", list(MISTAKES))
def test_state_mistakes_are_caught(mistake):
    """each mistake moves the output by many orders of magnitude more than the tolerance"""
    cfg, pad, sb, w, c = _setup("melgan_causal_mb")
    ref = _delayed(RS.whole_utterance(w, c, cfg, pad, sb), sb)
    first = min_first_frames(cfg, pad)
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        assert _err(RS.stream(w, c, cfg, schedule, pad, sb, first=first), ref) <= TOL
        assert _err(RS.stream(w, c, cfg, schedule, pad, sb, first=first, **MISTAKES[mistake]), ref) > 1e6 * TOL, (mistake, schedule)
