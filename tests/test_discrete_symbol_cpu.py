"""Discrete-symbol HiFi-GAN generators without a GPU: the CPU oracle against the reference's golden outputs, and the
mirror's module structure (state-dict names and shapes, weight-norm round trip, the reference's failing
configurations, loading by config name) against the reference's."""
import pytest
import torch

from helpers import ORACLE_TOL, golden_effective_weights, golden_weights, load_golden, rel_l2
from oracle import ref_discrete

GEN = ["dsym_small", "dsym_vctk"]
DUR = ["dsym_dur_cvss", "dsym_dur_odd"]


def _cls(meta):
    from parallelwavegan_b200 import models

    return {"dsym_generator": models.DiscreteSymbolHiFiGANGenerator,
            "dsym_duration_generator": models.DiscreteSymbolDurationGenerator}[meta["kind"]]


def _weights(meta, fold=True):
    w = golden_effective_weights(meta) if fold else golden_weights(meta)
    if "linear_bias" in meta:
        w["duration_predictor.linear.bias"] = torch.full_like(w["duration_predictor.linear.bias"], meta["linear_bias"])
        w["duration_predictor.linear.weight"] = w["duration_predictor.linear.weight"] * meta["linear_weight_scale"]
    return w


@pytest.mark.parametrize("name", GEN)
def test_oracle_matches_reference_generator(name):
    meta, g = load_golden(name)
    w, cfg, c = _weights(meta), meta["kwargs"], g["c"]
    with torch.no_grad():
        assert rel_l2(ref_discrete.dsym_generator(w, c, cfg), g["y"]) < ORACLE_TOL
        assert rel_l2(ref_discrete.dsym_generator(w, c[:1], cfg)[0].t(), g["y_inf"]) < ORACLE_TOL
        if "y_inf_g" in g:
            cg = c[:1].clone()
            cg[:, 1] = meta["g"]
            assert rel_l2(ref_discrete.dsym_generator(w, cg, cfg)[0].t(), g["y_inf_g"]) < ORACLE_TOL


@pytest.mark.parametrize("name", DUR)
def test_oracle_matches_reference_duration(name):
    meta, g = load_golden(name)
    w, cfg, c = _weights(meta), meta["kwargs"], g["c"]
    with torch.no_grad():
        y, ds_out = ref_discrete.dsym_duration_forward(w, c, g["ds"].clone(), cfg)
        assert rel_l2(y, g["y"]) < ORACLE_TOL and rel_l2(ds_out, g["ds_out"]) < ORACLE_TOL
        y_syn, ds_syn = ref_discrete.dsym_duration_synthesis(w, c, cfg)
        assert torch.equal(ds_syn, g["ds_syn"])
        assert rel_l2(y_syn, g["y_syn"]) < ORACLE_TOL
        y0, _ = ref_discrete.dsym_duration_synthesis(w, c[:1], cfg)
        assert rel_l2(y0[0].t(), g["y_inf"]) < ORACLE_TOL
        y0, _ = ref_discrete.dsym_duration_forward(w, c[:1], g["ds"][:1].clone(), cfg)
        assert rel_l2(y0[0].t(), g["y_inf_ds"]) < ORACLE_TOL
    assert int(g["ds_syn"].min()) == 0 and int(g["ds_syn"].max()) >= 2
    assert int(c[1, 0, -1]) == cfg["num_embs"] and int(g["ds"][1, -1]) == 0  # the padded symbol


def test_length_regulator_zero_rule_in_place():
    e = torch.randn(3, 4, 5)
    ds = torch.zeros(3, 5, dtype=torch.int64)
    y = ref_discrete.length_regulate(e, ds)
    assert torch.equal(ds, torch.ones(3, 5, dtype=torch.int64)) and torch.equal(y, e)
    ds = torch.tensor([[0, 0], [1, 2]])
    y = ref_discrete.length_regulate(e[:2, :, :2], ds)
    assert torch.equal(ds, torch.tensor([[0, 0], [1, 2]])) and y.shape == (2, 4, 3) and not y[0].any()


@pytest.mark.parametrize("name", GEN + DUR)
def test_state_dict_matches_reference(name):
    meta, _ = load_golden(name)
    m = _cls(meta)(**meta["kwargs"])
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == [(k, list(s)) for k, s in meta["spec"]]
    m.load_state_dict(golden_weights(meta), strict=True)
    m.remove_weight_norm()
    folded = []
    for k, s in meta["spec"]:
        if k.endswith(".weight_g"):
            continue
        folded.append((k[: -len("_v")] if k.endswith(".weight_v") else k, list(s)))
    assert sorted((k, list(v.shape)) for k, v in m.state_dict().items()) == sorted(folded)
    m.apply_weight_norm()
    keys = sorted(k for k, _ in meta["spec"])
    if meta["kind"] == "dsym_duration_generator":  # apply_weight_norm now reaches the predictor convs, as in the reference
        keys = sorted(k for k, _ in meta["spec"] if not (k.startswith("duration_predictor.conv.") and k.endswith(".0.weight")))
        keys = sorted(keys + [k[: -len("weight")] + s for k, _ in meta["spec"]
                              if k.startswith("duration_predictor.conv.") and k.endswith(".0.weight") for s in ("weight_g", "weight_v")])
    assert sorted(m.state_dict()) == keys


def test_state_dict_loads_reference_spec_without_weight_norm():
    meta, _ = load_golden("dsym_small")
    m = _cls(meta)(**dict(meta["kwargs"], use_weight_norm=False))
    m.load_state_dict(golden_effective_weights(meta))
    assert not hasattr(m, "register_stats")


def test_duration_predictor_is_not_weight_normed():
    meta, _ = load_golden("dsym_dur_cvss")
    keys = [k for k, _ in meta["spec"] if k.startswith("duration_predictor.")]
    assert keys == ["duration_predictor.conv.0.0.weight", "duration_predictor.conv.0.0.bias", "duration_predictor.conv.0.2.weight",
                    "duration_predictor.conv.0.2.bias", "duration_predictor.conv.1.0.weight", "duration_predictor.conv.1.0.bias",
                    "duration_predictor.conv.1.2.weight", "duration_predictor.conv.1.2.bias", "duration_predictor.linear.weight",
                    "duration_predictor.linear.bias"]


def test_reference_failures_raise_at_forward():
    """concat_spk_emb=True and duration-with-speakers construct (same state dict as the reference) but fail at forward,
    as the reference does (verified there): both raise a RuntimeError before any launch."""
    from parallelwavegan_b200 import models

    meta, _ = load_golden("dsym_small")
    kw = dict(meta["kwargs"], num_spk_embs=4, spk_emb_dim=16, concat_spk_emb=True)
    m = models.DiscreteSymbolHiFiGANGenerator(**kw)
    assert m.input_conv.in_channels == kw["in_channels"] + 16
    with pytest.raises(RuntimeError, match="concat_spk_emb"):
        m(torch.zeros(1, 2, 5))
    meta, _ = load_golden("dsym_dur_odd")
    kw = dict(meta["kwargs"], num_spk_embs=3, spk_emb_dim=meta["kwargs"]["in_channels"])
    m = models.DiscreteSymbolDurationGenerator(**kw)
    for call in (lambda: m(torch.zeros(1, 2, 5), torch.ones(1, 5, dtype=torch.int64)), lambda: m.synthesis(torch.zeros(1, 2, 5))):
        with pytest.raises(RuntimeError, match="duration predictor expects"):
            call()


def test_getattr_and_load_model(tmp_path):
    from parallelwavegan_b200 import models, utils

    for name in ("DiscreteSymbolHiFiGANGenerator", "DiscreteSymbolDurationGenerator"):
        assert getattr(models, name) is getattr(models, name)
    for fixture, gtype in (("dsym_vctk", "DiscreteSymbolHiFiGANGenerator"), ("dsym_dur_odd", "DiscreteSymbolDurationGenerator")):
        meta, _ = load_golden(fixture)
        sd = golden_weights(meta)
        path = tmp_path / f"{fixture}.pkl"
        torch.save({"model": {"generator": sd}}, path)
        m = utils.load_model(str(path), config={"generator_type": gtype, "generator_params": meta["kwargs"], "format": "npy"})
        assert type(m) is getattr(models, gtype)
        assert all(torch.equal(m.state_dict()[k], v) for k, v in sd.items())


def test_duration_collater_rejects_what_the_reference_rejects():
    from parallelwavegan_b200 import datasets

    for kw in (dict(use_aux_input=False), dict(use_noise_input=True)):
        with pytest.raises(RuntimeError, match="use_duration"):
            datasets.Collater(use_duration=True, **kw)
