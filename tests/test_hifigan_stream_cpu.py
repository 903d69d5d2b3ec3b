"""Streaming a causal HiFi-GAN, on the CPU: the chunked oracle (oracle/ref_hifigan_stream.py) equals the whole-utterance
causal generator in float64 for every chunk schedule, reproduces the golden ``inference`` output of the real reference,
and each plausible state mistake breaks that equality."""
import json

import pytest
import torch

from helpers import ORACLE_TOL, golden_effective_weights, load_golden, rel_l2
from oracle import ref_hifigan_stream as RS
from oracle import synth
from oracle.ref_ops import fold_weight_norm

# one frame at a time, chunks shorter and longer than the deepest history (the level input's 10 samples and the
# output conv's 6 are below a frame of the finest level; the 6-frame input-conv history is the deepest in frames), and an
# irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
TOL = 1e-12
SMALL = dict(in_channels=80, out_channels=1, channels=32, kernel_size=7, upsample_scales=[8, 8, 2, 2],
             upsample_kernel_sizes=[16, 16, 4, 4], resblock_kernel_sizes=[3, 7, 11], resblock_dilations=[[1, 3, 5]] * 3,
             use_causal_conv=True)
CONFIGS = {
    "no_additional_convs": dict(SMALL, use_additional_convs=False),
    # ReLU, irregular kernel sizes and dilations, odd scales
    "relu_irregular": dict(SMALL, kernel_size=5, upsample_scales=[5, 3, 2], upsample_kernel_sizes=[10, 6, 4],
                           resblock_kernel_sizes=[5, 9], resblock_dilations=[[1, 2], [2, 3, 7]], nonlinear_activation="ReLU",
                           nonlinear_activation_params={}),
}


def _cfg(kw):
    slope = 0.0 if kw.get("nonlinear_activation") == "ReLU" else kw.get("nonlinear_activation_params", {}).get("negative_slope", 0.1)
    return dict(kw, negative_slope=slope)


def _setup(name):
    """(cfg, float64 effective weights, c (2, 80, T) float64) of the golden model or a synthetic config"""
    if name == "hifigan_causal":
        meta, _ = load_golden(name)
        w = golden_effective_weights(meta)
        return _cfg(meta["kwargs"]), {k: v.double() for k, v in w.items()}, synth.randn(meta["c_shape"], meta["c_seed"]).double()
    from parallelwavegan_b200 import models

    kw = CONFIGS[name]
    m = models.HiFiGANGenerator(**json.loads(json.dumps(kw)))
    sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 21, 1.15)
    return _cfg(kw), {k: v.double() for k, v in fold_weight_norm(sd).items()}, synth.randn((2, 80, 19), 22).double()


def _err(y, ref):
    return float((y - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("name", ["hifigan_causal", *CONFIGS])
def test_chunked_oracle_equals_whole_utterance(name, schedule):
    cfg, w, c = _setup(name)
    ref = RS.whole_utterance(w, c, cfg)
    y = RS.stream(w, c, cfg, SCHEDULES[schedule])
    assert y.shape == ref.shape
    assert _err(y, ref) <= TOL, _err(y, ref)


def test_chunked_oracle_reproduces_golden_inference():
    meta, g = load_golden("hifigan_causal")
    cfg, w, c = _setup("hifigan_causal")
    y = RS.stream({k: v.float() for k, v in w.items()}, c[:1].float(), cfg, SCHEDULES["mixed"], dtype=torch.float32)
    assert rel_l2(y[0].t(), g["y_inf"]) < ORACLE_TOL


@pytest.mark.parametrize("mistake", ["dil_short", "up_zero", "lvl_first_only"])
@pytest.mark.parametrize("name", ["hifigan_causal", "relu_irregular"])
def test_state_mistakes_are_caught(name, mistake):
    """each mistake moves the output by many orders of magnitude more than the tolerance"""
    cfg, w, c = _setup(name)
    kw = {"dil_short": dict(dil_short=1), "up_zero": dict(up_zero=True), "lvl_first_only": dict(lvl_first_only=True)}[mistake]
    ref = RS.whole_utterance(w, c, cfg)
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        assert _err(RS.stream(w, c, cfg, schedule), ref) <= TOL
        assert _err(RS.stream(w, c, cfg, schedule, **kw), ref) > 1e6 * TOL, (mistake, schedule)
