"""Streaming a causal Parallel WaveGAN, on the CPU: the chunked oracle (oracle/ref_pwg_stream.py) equals the
whole-utterance causal generator in float64 for every chunk schedule, reproduces the golden ``inference`` outputs of
the real reference, and each plausible state mistake breaks that equality."""
import math

import pytest
import torch

from helpers import ORACLE_TOL, golden_effective_weights, load_golden, rel_l2
from oracle import ref_pwg_stream as RS
from oracle import synth

GENERATORS = ["pwg_causal_small_acw0", "pwg_causal_small_acw1", "pwg_causal_small_acw2", "pwg_causal_small_acw3",
              "pwg_causal_small_upnet", "pwg_causal_v1", "pwg_causal_k2"]
# one frame at a time, chunks shorter and longer than the largest layer history (v1: 2048 samples = 8 frames of 256),
# and an irregular mix
SCHEDULES = {"ones": [1], "short": [3], "long": [17], "mixed": [1, 7, 2, 33, 5, 1, 12]}
TOL = 1e-12


def _setup(name):
    meta, g = load_golden(name)
    kw = meta["kwargs"]
    cfg = dict(kw, upsample_scales=kw["upsample_params"]["upsample_scales"])
    w = {k: v.double() for k, v in golden_effective_weights(meta).items()}
    ctx = kw["aux_context_window"]
    c = synth.randn(meta["c_shape"], meta["c_seed"])
    z = synth.randn(meta["z_shape"], meta["z_seed"])
    return meta, g, cfg, w, c[:, :, ctx: c.shape[-1] - ctx].double(), z.double()


def _err(y, ref):
    return float((y - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("name", GENERATORS)
def test_chunked_oracle_equals_whole_utterance(name, schedule):
    _, _, cfg, w, c, z = _setup(name)
    ref = RS.whole_utterance(w, z, c, cfg)
    y = RS.stream(w, z, c, cfg, SCHEDULES[schedule])
    assert y.shape == ref.shape
    assert _err(y, ref) <= TOL, _err(y, ref)


@pytest.mark.parametrize("name", GENERATORS)
def test_chunked_oracle_reproduces_golden_inference(name):
    _, g, cfg, w, c, z = _setup(name)
    y = RS.stream({k: v.float() for k, v in w.items()}, z[:1].float(), c[:1].float(), cfg, SCHEDULES["mixed"], dtype=torch.float32)
    assert rel_l2(y[0].t(), g["y_inf"]) < ORACLE_TOL


@pytest.mark.parametrize("mistake", ["wn_short", "cin_zero", "fir_one_frame"])
@pytest.mark.parametrize("name", ["pwg_causal_small_acw2", "pwg_causal_v1", "pwg_causal_k2"])
def test_state_mistakes_are_caught(name, mistake):
    """each mistake moves the output by many orders of magnitude more than the tolerance"""
    _, _, cfg, w, c, z = _setup(name)
    kw = {"wn_short": dict(wn_short=1), "cin_zero": dict(cin_init="zero"), "fir_one_frame": dict(fir_frames=1)}[mistake]
    ref = RS.whole_utterance(w, z, c, cfg)
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        assert _err(RS.stream(w, z, c, cfg, schedule), ref) <= TOL
        assert _err(RS.stream(w, z, c, cfg, schedule, **kw), ref) > 1e6 * TOL, (mistake, schedule)


def test_schedules_cover_the_history_lengths():
    """the schedules include chunks shorter and longer than the largest layer history of PWG v1"""
    meta, _ = load_golden("pwg_causal_v1")
    kw = meta["kwargs"]
    hop = math.prod(kw["upsample_params"]["upsample_scales"])
    lps = kw["layers"] // kw["stacks"]
    hmax = (kw["kernel_size"] - 1) * 2 ** (lps - 1)
    sizes = [n * hop for s in SCHEDULES.values() for n in s]
    assert min(sizes) < hmax < max(sizes)
