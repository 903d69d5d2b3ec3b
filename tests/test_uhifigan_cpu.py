"""UHiFiGAN generator without a GPU: the CPU oracle against the reference's golden outputs, and the mirror's
module structure (state-dict names and shapes, constructor behaviour) against the reference's."""
import pytest
import torch

from helpers import ORACLE_TOL, golden_effective_weights, load_golden, rel_l2
from oracle import synth
from oracle.ref_uhifigan import uhifigan_generator

NAMES = ["uhifigan_small", "uhifigan_opencpop", "uhifigan_odd"]


def golden_inputs(meta):
    c = synth.randn(tuple(meta["c_shape"]), meta["c_seed"])
    f0 = synth.randn(tuple(meta["f0_shape"]), meta["f0_seed"])
    e = synth.randn(tuple(meta["e_shape"]), meta["e_seed"], meta["e_scale"])
    return c, f0, e


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    meta, g = load_golden(name)
    w = golden_effective_weights(meta)
    c, _, e = golden_inputs(meta)
    with torch.no_grad():
        y = uhifigan_generator(w, e, c, meta["kwargs"])
        y0 = uhifigan_generator(w, e[:1], c[:1], meta["kwargs"])
    assert tuple(y.shape) == tuple(g["y"].shape)
    assert rel_l2(y, g["y"]) < ORACLE_TOL
    assert rel_l2(y0[0].t(), g["y_inf"]) < ORACLE_TOL


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_matches_reference(name):
    from parallelwavegan_b200 import models

    meta, _ = load_golden(name)
    m = models.UHiFiGANGenerator(**meta["kwargs"])
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == [(k, list(s)) for k, s in meta["spec"]]
    m.remove_weight_norm()
    folded = []
    for k, s in meta["spec"]:
        if k.endswith(".weight_g"):
            continue
        folded.append((k[: -len("_v")] if k.endswith(".weight_v") else k, list(s)))
    assert sorted((k, list(v.shape)) for k, v in m.state_dict().items()) == sorted(folded)
    m.apply_weight_norm()
    assert sorted(m.state_dict()) == sorted(k for k, _ in meta["spec"])


def test_state_dict_loads_reference_spec_without_weight_norm():
    from parallelwavegan_b200 import models

    meta, _ = load_golden("uhifigan_small")
    m = models.UHiFiGANGenerator(**dict(meta["kwargs"], use_weight_norm=False))
    m.load_state_dict(golden_effective_weights(meta))


def test_causal_raises_type_error():
    from parallelwavegan_b200 import models

    meta, _ = load_golden("uhifigan_small")
    with pytest.raises(TypeError):
        models.UHiFiGANGenerator(**dict(meta["kwargs"], use_causal_conv=True))


def test_getattr_by_config_name():
    from parallelwavegan_b200 import models

    assert getattr(models, "UHiFiGANGenerator") is models.UHiFiGANGenerator
