"""Causal Parallel WaveGAN and ResidualParallelWaveGANDiscriminator on the CPU: the oracle restatement
(oracle/ref_causal_pwg.py) reproduces the golden vectors of the real reference, the mirrors' state dicts match the
reference's names and shapes, and construction accepts the causal and dropout variants."""
import json

import pytest
import torch

from helpers import ORACLE_TOL, golden_effective_weights, load_golden, rel_l2
from oracle import ref_causal_pwg, synth

GENERATORS = ["pwg_causal_small_acw0", "pwg_causal_small_acw1", "pwg_causal_small_acw2", "pwg_causal_small_acw3",
              "pwg_causal_small_upnet", "pwg_causal_v1", "pwg_causal_k2", "pwg_causal_melgan_up"]
DISCRIMINATORS = ["rpwgd_default", "rpwgd_causal", "rpwgd_small"]
RPWGD_DEFAULTS = dict(layers=30, stacks=3, kernel_size=3)


def gen_cfg(kw):
    return dict(kw, upsample_scales=kw["upsample_params"]["upsample_scales"])


@pytest.mark.parametrize("name", GENERATORS)
def test_oracle_reproduces_causal_generator_golden(name):
    meta, g = load_golden(name)
    w = golden_effective_weights(meta)
    c = synth.randn(meta["c_shape"], meta["c_seed"])
    z = synth.randn(meta["z_shape"], meta["z_seed"])
    cfg = gen_cfg(meta["kwargs"])
    with torch.no_grad():
        y = ref_causal_pwg.pwg_generator(w, z, c, cfg)
        c_up = ref_causal_pwg.pwg_upsample_net(w, c, cfg)
    assert tuple(y.shape) == tuple(g["y"].shape)
    assert rel_l2(y, g["y"]) < ORACLE_TOL
    assert rel_l2(c_up[:, :, :512], g["c_up"]) < ORACLE_TOL


@pytest.mark.parametrize("name", DISCRIMINATORS)
def test_oracle_reproduces_residual_discriminator_golden(name):
    meta, g = load_golden(name)
    w = golden_effective_weights(meta)
    x = synth.randn(meta["x_shape"], meta["x_seed"], meta["x_scale"])
    with torch.no_grad():
        y = ref_causal_pwg.residual_pwg_discriminator(w, x, dict(RPWGD_DEFAULTS, **meta["kwargs"]))
    assert rel_l2(y, g["final0"]) < ORACLE_TOL


def test_oracle_centred_matches_ref_ops():
    """with every flag at its default the restatement is the existing centred PWG oracle"""
    from oracle import ref_ops

    meta, g = load_golden("pwg_small")
    w = golden_effective_weights(meta)
    c = synth.randn(meta["c_shape"], meta["c_seed"])
    z = synth.randn(meta["z_shape"], meta["z_seed"])
    cfg = gen_cfg(meta["kwargs"])
    assert rel_l2(ref_causal_pwg.pwg_generator(w, z, c, cfg), ref_ops.pwg_generator(w, z, c, cfg)) < ORACLE_TOL


@pytest.mark.parametrize("name", GENERATORS + DISCRIMINATORS)
def test_mirror_state_dict_spec(name):
    from parallelwavegan_b200 import models

    meta, _ = load_golden(name)
    cls = models.ResidualParallelWaveGANDiscriminator if name.startswith("rpwgd") else models.ParallelWaveGANGenerator
    m = cls(**json.loads(json.dumps(meta["kwargs"])))
    assert [(k, list(v.shape)) for k, v in m.state_dict().items()] == [(k, list(s)) for k, s in meta["spec"]]
    m.remove_weight_norm()
    assert not any(k.endswith("weight_g") for k in m.state_dict())


def test_causal_and_dropout_construction():
    from parallelwavegan_b200 import layers, models

    blk = layers.WaveNetResidualBlock(kernel_size=2, dropout=0.05, use_causal_conv=True)
    assert blk.conv.padding == (1,) and blk.use_causal_conv
    with pytest.raises(AssertionError):
        layers.WaveNetResidualBlock(kernel_size=2)  # even kernels only as causal convs
    up = layers.ConvInUpsampleNetwork([4, 4], aux_channels=10, aux_context_window=2, use_causal_conv=True)
    assert up.conv_in.kernel_size == (3,) and up.use_causal_conv and up.upsample.use_causal_conv
    up0 = layers.ConvInUpsampleNetwork([4, 4], aux_channels=10, aux_context_window=0, use_causal_conv=True)
    assert not up0.use_causal_conv and up0.upsample.use_causal_conv  # the reference's aux_context_window = 0 quirk
    assert up0.upsample.up_layers[1].padding == (0, 8)
    models.ParallelWaveGANGenerator(use_causal_conv=True, layers=6, stacks=3)
    models.ResidualParallelWaveGANDiscriminator(layers=6, stacks=3, use_causal_conv=True, dropout=0.1)


def test_unsupported_upsampler_variants_still_raise():
    from parallelwavegan_b200 import layers
    from parallelwavegan_b200.capi import PwgbError

    with pytest.raises(PwgbError):
        layers.UpsampleNetwork([4, 4], nonlinear_activation="ReLU", use_causal_conv=True)
    with pytest.raises(PwgbError):
        layers.UpsampleNetwork([4, 4], freq_axis_kernel_size=3, use_causal_conv=True)
