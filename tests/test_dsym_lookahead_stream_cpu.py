"""Streaming a discrete-symbol HiFi-GAN with a fixed lookahead, on the CPU: the chunked oracle
(oracle/ref_dsym_lookahead_stream.py) followed by its flush equals [zeros(delay) | the whole-utterance generator] in
float64 for every chunk schedule, with and without speakers, its delay is the lookahead of the recipes' shapes, and
taking the speaker from each chunk instead of latching the first frame's breaks that equality."""
import json

import pytest
import torch

from helpers import golden_effective_weights, load_golden
from oracle import ref_dsym_lookahead_stream as RD
from oracle import synth
from oracle.ref_ops import fold_weight_norm

SCHEDULES = {"ones": [1], "short": [3], "long": [7], "mixed": [1, 4, 2, 9, 1, 3]}
TOL = 1e-12
# the 24 kHz recipes' upsampling (hop 480) on few channels
SYN24 = dict(in_channels=32, out_channels=1, channels=64, num_embs=50, num_spk_embs=4, spk_emb_dim=32, kernel_size=7,
             upsample_scales=[12, 10, 2, 2], upsample_kernel_sizes=[24, 20, 4, 4], resblock_kernel_sizes=[3, 7, 11],
             resblock_dilations=[[1, 3, 5]] * 3)


def _setup(name, frames=None):
    """(cfg, float64 effective weights, c (B, K, T) int64) of a golden model or of ``syn24``; with speakers, every frame
    of c gets a different speaker id, of which only the first may count"""
    if name == "syn24":
        from parallelwavegan_b200 import models

        m = models.DiscreteSymbolHiFiGANGenerator(**json.loads(json.dumps(SYN24)))
        sd = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 31, 1.15)
        cfg, w = SYN24, fold_weight_norm(sd)
        g = torch.Generator().manual_seed(5)
        c = torch.stack([torch.randint(0, cfg["num_embs"], (2, frames or 11), generator=g),
                         torch.randint(0, cfg["num_spk_embs"], (2, frames or 11), generator=g)], 1)
    else:
        meta, gold = load_golden(name)
        cfg, w = meta["kwargs"], golden_effective_weights(meta)
        c = gold["c"].long()[..., :frames] if frames else gold["c"].long()
        if cfg.get("num_spk_embs", 128) > 0:
            c = c.clone()
            c[:, 1] = torch.arange(c.shape[-1]) % cfg["num_spk_embs"]
            c[1, 1] = c[1, 1].flip(-1)
    return cfg, {k: v.double() for k, v in w.items()}, c


def _expected(w, c, cfg, delay):
    ref = RD.whole_utterance(w, c, cfg)
    return torch.cat([ref.new_zeros(ref.shape[:-1] + (delay,)), ref], -1)


def _err(y, ref):
    return float((y - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("name", ["dsym_small", "dsym_vctk", "syn24"])
def test_chunked_oracle_equals_whole_utterance(name, schedule):
    cfg, w, c = _setup(name, 10 if name == "dsym_vctk" else None)
    delay = RD.DSymLookaheadRef(w, cfg).delay
    ref = _expected(w, c, cfg, delay)
    y = RD.stream(w, c, cfg, SCHEDULES[schedule])
    assert y.shape == ref.shape
    assert _err(y, ref) <= TOL, _err(y, ref)


@pytest.mark.parametrize("frames", [1, 2])
def test_utterances_shorter_than_the_delay(frames):
    cfg, w, c = _setup("dsym_vctk", frames)
    ref = RD.DSymLookaheadRef(w, cfg)
    assert frames * ref.hop < ref.delay
    assert _err(RD.stream(w, c, cfg, [1]), _expected(w, c, cfg, ref.delay)) <= TOL


@pytest.mark.parametrize("name, delay", [("dsym_vctk", 3482), ("syn24", 4526), ("dsym_small", 212)])
def test_delay_of_the_recipes_shapes(name, delay):
    """3482 samples for the 16 kHz recipes' scales (10, 8, 2, 2) and 4526 for the 24 kHz ones (12, 10, 2, 2)"""
    cfg, w, _ = _setup(name)
    assert RD.DSymLookaheadRef(w, cfg).delay == delay


@pytest.mark.parametrize("name", ["dsym_vctk", "syn24"])
def test_chunk_speaker_is_caught(name):
    """the whole utterance adds the first frame's speaker to every frame: a stream that reads each chunk's first frame
    differs as soon as a later chunk starts on another speaker id"""
    cfg, w, c = _setup(name, 6)
    delay = RD.DSymLookaheadRef(w, cfg).delay
    ref = _expected(w, c, cfg, delay)
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        assert _err(RD.stream(w, c, cfg, schedule), ref) <= TOL
        assert _err(RD.stream(w, c, cfg, schedule, chunk_speaker=True), ref) > 1e6 * TOL, schedule


# ---------------------------------------------------------------------------------------------------- duration model
def _dur_setup(name="dsym_dur_cvss", item=0):
    """(cfg, float64 effective weights (the fixture's predictor bias and scale applied), symbols (S,) of one item)"""
    meta, gold = load_golden(name)
    w = golden_effective_weights(meta)
    if "linear_bias" in meta:
        w["duration_predictor.linear.bias"] = torch.full_like(w["duration_predictor.linear.bias"], meta["linear_bias"])
        w["duration_predictor.linear.weight"] = w["duration_predictor.linear.weight"] * meta["linear_weight_scale"]
    return meta["kwargs"], {k: v.double() for k, v in w.items()}, gold["c"].long()[item, 0], gold


def _dur_expected(w, c, cfg, delay):
    from oracle.ref_discrete import dsym_duration_synthesis

    y, ds = dsym_duration_synthesis(w, c.view(1, 1, -1), cfg)
    return torch.cat([y.new_zeros(y.shape[:-1] + (delay,)), y], -1), ds[0]


@pytest.mark.parametrize("schedule", list(SCHEDULES))
@pytest.mark.parametrize("item", [0, 1])
def test_duration_oracle_equals_synthesis(item, schedule):
    cfg, w, c, gold = _dur_setup(item=item)
    ref = RD.DSymDurationLookaheadRef(w, cfg)
    assert ref.P == 2
    exp, ds = _dur_expected(w, c, cfg, ref.delay)
    assert torch.equal(ds, gold["ds_syn"][item])
    y, d, _ = RD.duration_stream(w, c, cfg, SCHEDULES[schedule])
    assert torch.equal(d, ds)
    assert y.shape == exp.shape and _err(y, exp) <= TOL, _err(y, exp)


def test_duration_oracle_all_zero_rule():
    """a predictor whose every duration rounds to 0: the item alone gets unit durations, as synthesis of a batch of one"""
    cfg, w, c, _ = _dur_setup()
    w = dict(w)
    w["duration_predictor.linear.bias"] = torch.full_like(w["duration_predictor.linear.bias"], -30.0)
    ref = RD.DSymDurationLookaheadRef(w, cfg)
    exp, ds = _dur_expected(w, c, cfg, ref.delay)
    assert int(ds.sum()) == len(c)
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        y, d, _ = RD.duration_stream(w, c, cfg, schedule)
        assert int(d.sum()) == 0 and _err(y, exp) <= TOL


@pytest.mark.parametrize("mistake", ["look", "ln_unmasked", "zero_rule_per_chunk", "restart_runs", "flush_no_tail"])
def test_duration_mistakes_are_caught(mistake):
    """each mistake changes the durations, moves their log-domain values or moves the audio by many orders of magnitude
    more than the tolerance (a wrong lookahead may leave the rounded durations of this fixture intact)"""
    from oracle.ref_discrete import duration_predictor, embed

    cfg, w, c, _ = _dur_setup()
    if mistake == "restart_runs":  # runs of several frames, so that body pushes cut them
        w = dict(w, **{"duration_predictor.linear.bias": w["duration_predictor.linear.bias"] + 1.0})
    kw = {"look": 1} if mistake == "look" else {mistake: True}
    exp, ds = _dur_expected(w, c, cfg, RD.DSymDurationLookaheadRef(w, cfg).delay)
    x = duration_predictor(w, embed(w, c.view(1, 1, -1), cfg), cfg)[0]
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        y, d, xs = RD.duration_stream(w, c, cfg, schedule)
        assert torch.equal(d, ds) and _err(y, exp) <= TOL and _err(xs, x) <= TOL
    caught = []
    for schedule in (SCHEDULES["ones"], SCHEDULES["mixed"]):
        y, d, xs = RD.duration_stream(w, c, cfg, schedule, **kw)
        caught.append(not torch.equal(d, ds) or y.shape != exp.shape or _err(y, exp) > 1e6 * TOL
                      or xs.shape != x.shape or _err(xs, x) > 1e6 * TOL)
    assert any(caught), mistake
